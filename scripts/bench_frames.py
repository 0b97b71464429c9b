"""Device time per step of the two-call frame path, FastBaseTransform()(frames) + Yolact.infer_padded, against the fused
Yolact.infer_frames (FastBaseTransform inside the stem's operand loader), on yolact_base from uint8 BGR frames to 550^2.

Both paths run on the same net and are alternated in one process, one timed window each per round, so that clock and
neighbour drift hits both alike; the table gives the median over rounds.  Prints the GPU name and power limit, which
belong with every number.

    python scripts/bench_frames.py [--precision f16x3] [--rounds 5] [--steps 20]
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


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def window_ms(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="f16x3", choices=["f16x3", "f16tc", "f32"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_frames measures on the GPU; there is no CPU fallback"

    cfg = CONFIGS["yolact_base_config"].copy()
    yolact_b200.cfg.replace(cfg.copy())
    net = yolact_b200.Yolact(cfg, precision=a.precision)
    net.detect.use_fast_nms = True
    net.load_state_dict(deterministic_state_dict(net.state_dict(), 0))
    net.eval()
    xf = FastBaseTransform(net.cfg)
    rng = np.random.RandomState(0)

    print("# %s; yolact_base %s, uint8 BGR frames -> %d^2" % (gpu_info(), a.precision, cfg.max_size))
    print("| batch | frame | two-call ms/step | fused ms/step | fused / two-call | identical |")
    print("|---|---|---|---|---|---|")
    for B in (1, 8):
        for h, w in ((720, 1280), (480, 640)):
            f = torch.from_numpy(rng.randint(0, 256, size=(B, h, w, 3)).astype(np.uint8)).cuda()
            two = lambda: net.infer_padded(xf(f))
            fused = lambda: net.infer_frames(f)
            for _ in range(a.warmup):   # eager, capture, replay of both graphs
                two()
                fused()
            torch.cuda.synchronize()
            same = all(torch.equal(p, q) for p, q in zip(two()[:5], fused()[:5]))
            t2, tf = [], []
            for _ in range(a.rounds):
                t2.append(window_ms(two, a.steps))
                tf.append(window_ms(fused, a.steps))
            m2, mf = statistics.median(t2), statistics.median(tf)
            print("| %d | %dx%d | %.3f (%.3f-%.3f) | %.3f (%.3f-%.3f) | %.3f | %s |" % (
                B, h, w, m2, min(t2), max(t2), mf, min(tf), max(tf), mf / m2, same), flush=True)


if __name__ == "__main__":
    main()
