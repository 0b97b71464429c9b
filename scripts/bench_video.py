"""Time per frame of eval.py's video display loop on the GPU side: uint8 BGR frames -> drawn frames -> host, 8 frames per
step, for three routes:

  (a) forward_frames + today's eval.py display per frame: postprocess (fp32 masks of every row at frame size, with
      rescore_bbox), argsort, the top_k gather, .cpu() of classes / scores / boxes, the reference's torch blend
      (eval.py:189-209) and `(img_gpu * 255).byte().cpu()`;
  (b) forward_frames + render_masks on the step's 8 frames, then the images to the host;
  (c) render_frames with two steps in flight: step i+1 is enqueued before the host waits for step i's images, which is
      possible because render_frames never syncs the host.

yolact_base with deterministic weights at 550^2 input, seeded frames of 550x550 and 1080x1920, top_k 5, score_threshold
0.  The routes alternate, one window of --steps steps each per round, each window ending in a device synchronise; the
table gives the median over rounds of the host wall ms per frame and the CUDA-event ms per frame (events on the current
stream around the window), and whether (b) and (c) give identical images.  Prints the GPU name and power limit, which
belong with every number.

    python scripts/bench_video.py [--rounds 5] [--steps 4]
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
from yolact_b200.config import COLORS, CONFIGS
from yolact_b200.display import render_masks
from yolact_b200.output_utils import postprocess

TOP_K = 5


def reference_display(preds, frame, i):
    """eval.py:143-224 for image i with undo_transform=False, masks on, text drawn later from the host rows."""
    cfg = ybcfg.cfg
    img_gpu = frame.float() / 255.0
    save, cfg.rescore_bbox = cfg.rescore_bbox, True
    try:
        t = postprocess(preds, int(frame.shape[1]), int(frame.shape[0]), i)
    finally:
        cfg.rescore_bbox = save
    if t[1].numel() == 0:
        return (img_gpu * 255).byte().cpu().numpy()
    idx = t[1].argsort(0, descending=True)[:TOP_K]
    masks = t[3][idx]
    classes, scores, boxes = [x[idx].cpu().numpy() for x in t[:3]]
    n = min(TOP_K, classes.shape[0])
    if n > 0:
        masks = masks[:n, :, :, None]
        colors = torch.cat([(torch.tensor([COLORS[j * 5 % len(COLORS)][c] for c in (2, 1, 0)], dtype=torch.float32,
                                          device=frame.device) / 255.).view(1, 1, 1, 3) for j in range(n)], dim=0)
        masks_color = masks.repeat(1, 1, 1, 3) * colors * 0.45
        inv_alph_masks = masks * (-0.45) + 1
        masks_color_summand = masks_color[0]
        if n > 1:
            inv_alph_cumul = inv_alph_masks[:(n - 1)].cumprod(dim=0)
            masks_color_summand += (masks_color[1:] * inv_alph_cumul).sum(dim=0)
        img_gpu = img_gpu * inv_alph_masks.prod(dim=0) + masks_color_summand
    return (img_gpu * 255).byte().cpu().numpy()


def route_a(net, batches):
    out = []
    for frames in batches:
        preds = net.forward_frames(frames)
        out.append([reference_display(preds, frames[i], i) for i in range(frames.shape[0])])
    return out


def to_host(images):
    host = [im.to("cpu", non_blocking=True) for im in images]
    done = torch.cuda.Event()
    done.record()
    return host, done


def route_b(net, batches):
    out = []
    for frames in batches:
        images, _ = render_masks(net.forward_frames(frames), frames, top_k=TOP_K)
        host, done = to_host(images)
        done.synchronize()
        out.append(host)
    return out


def route_c(net, batches):
    out, pending = [], None
    for frames in batches:
        images, _ = net.render_frames(frames, top_k=TOP_K)
        nxt = to_host(images)
        if pending is not None:   # step i's images, while step i+1 runs
            pending[1].synchronize()
            out.append(pending[0])
        pending = nxt
    pending[1].synchronize()
    out.append(pending[0])
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
    ap.add_argument("--steps", type=int, default=4)
    args = ap.parse_args()
    print("GPU:", gpu_info())
    cfg = CONFIGS["yolact_base_config"].copy()
    yolact_b200.cfg.replace(cfg.copy())
    net = yolact_b200.Yolact(cfg, precision="f16x3")
    net.load_state_dict(deterministic_state_dict(net.state_dict(), 0))
    net.eval()
    B = 8
    print("| frames | route | wall ms / frame | event ms / frame | identical to (b) |")
    print("|---|---|---|---|---|")
    for (h, w) in ((550, 550), (1080, 1920)):
        g = torch.Generator().manual_seed(h * w)
        batches = [torch.randint(0, 256, (B, h, w, 3), generator=g, dtype=torch.uint8).cuda()
                   for _ in range(args.steps)]
        routes = {"(a) forward_frames + postprocess + torch blend": lambda: route_a(net, batches),
                  "(b) forward_frames + render_masks": lambda: route_b(net, batches),
                  "(c) render_frames, two steps in flight": lambda: route_c(net, batches)}
        results, times = {}, {k: [] for k in routes}
        for name, fn in routes.items():   # warm-up and the images
            fn()
            results[name] = window(fn)[2]
        for _ in range(args.rounds):
            for name, fn in routes.items():
                ev, wall, _ = window(fn)
                times[name].append((wall / (B * args.steps), ev / (B * args.steps)))
        ref = [im for step in results["(b) forward_frames + render_masks"] for im in step]
        for name in routes:
            got = [im for step in results[name] for im in step]
            if name.startswith("(a)"):
                same = "n/a (torch blend: +-1 truncation)"
            else:
                same = str(all(torch.equal(torch.as_tensor(a), b) for a, b in zip(got, ref)))
            wall = statistics.median(t[0] for t in times[name])
            ev = statistics.median(t[1] for t in times[name])
            print("| %dx%d | %s | %.3f | %.3f | %s |" % (h, w, name, wall, ev, same))


if __name__ == "__main__":
    main()
