"""Time per image of a folder of differently sized images (COCO-like sizes) through yolact_base at 550^2, three ways:

  (a) Yolact.infer_frames(f[None]) per image: batch 1, one call and one graph launch per image;
  (b) FastBaseTransform per image + torch.cat + Yolact.infer_padded at batch 8;
  (c) Yolact.infer_frames(list of 8 frames): one call and one graph whatever the sizes.

64 seeded uint8 BGR frames cycle through 16 sizes.  The paths are alternated in one process, one window (all 64 images)
each per round, so that clock and neighbour drift hits them alike; the table gives the median over rounds and the
range.  (b) and (c) must be bit-identical.  Prints the GPU name and power limit, which belong with every number.

    python scripts/bench_frame_list.py [--precision f16x3] [--rounds 5] [--batch 8]
"""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import yolact_b200
from oracle.weights import deterministic_state_dict
from yolact_b200.augmentations import FastBaseTransform
from yolact_b200.config import CONFIGS

# (h, w): common COCO val2017 image sizes
SIZES = [(480, 640), (640, 480), (427, 640), (375, 500), (612, 612), (424, 640), (640, 427), (500, 375),
         (426, 640), (640, 426), (333, 500), (500, 333), (360, 640), (480, 600), (512, 640), (640, 512)]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def window_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="f16x3", choices=["f16x3", "f16tc", "f32"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--images", type=int, default=64)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_frame_list measures on the GPU; there is no CPU fallback"
    assert a.images % a.batch == 0

    cfg = CONFIGS["yolact_base_config"].copy()
    yolact_b200.cfg.replace(cfg.copy())
    net = yolact_b200.Yolact(cfg, precision=a.precision)
    net.detect.use_fast_nms = True
    net.load_state_dict(deterministic_state_dict(net.state_dict(), 0))
    net.eval()
    xf = FastBaseTransform(net.cfg)
    rng = np.random.RandomState(0)
    frames = [torch.from_numpy(rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8)).cuda()
              for h, w in (SIZES[i % len(SIZES)] for i in range(a.images))]
    batches = [frames[i:i + a.batch] for i in range(0, a.images, a.batch)]

    def per_image():
        return [net.infer_frames(f[None]) for f in frames]

    def two_call():
        return [net.infer_padded(torch.cat([xf(f[None]) for f in fs])) for fs in batches]

    def frame_list():
        return [net.infer_frames(fs) for fs in batches]

    paths = [("(a) infer_frames(f[None]) per image", per_image),
             ("(b) FastBaseTransform per image + cat + infer_padded, B=%d" % a.batch, two_call),
             ("(c) infer_frames(list of %d)" % a.batch, frame_list)]
    for _, fn in paths:   # eager, capture, replay of every graph
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    same = all(torch.equal(p, q) for rb, rc in zip(two_call(), frame_list()) for p, q in zip(rb, rc) if p is not None)
    times = [[] for _ in paths]
    for _ in range(a.rounds):
        for t, (_, fn) in zip(times, paths):
            t.append(window_ms(fn) / a.images)

    print("# %s; yolact_base %s @%d, %d uint8 BGR frames cycling through %d sizes; median of %d alternated windows" % (
        gpu_info(), a.precision, cfg.max_size, a.images, len(SIZES), a.rounds))
    print("| path | ms / image (range) | vs (b) |")
    print("|---|---|---|")
    mb = statistics.median(times[1])
    for (name, _), t in zip(paths, times):
        m = statistics.median(t)
        print("| %s | %.3f (%.3f-%.3f) | %.3f |" % (name, m, min(t), max(t), m / mb))
    print("(b) and (c) bit-identical: %s" % same, flush=True)


if __name__ == "__main__":
    main()
