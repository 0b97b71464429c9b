"""Frames/s of eval.py's evalvideo network stage under DataParallel, for 1..N GPUs:

    imgs = torch.nn.DataParallel(FastBaseTransform())(torch.stack(frames, 0))     # eval.py:662,692-695
    preds = CustomDataParallel(net)(imgs)                                          # eval.py:630-634,661,697-707

with --video_multiframe frames per step at 1, N and 2N (evalvideo's frames arrive on cuda:0 as float BGR, as
transform_frame's `.cuda().float()` leaves them; the disk read and that host-to-device copy are not timed).  On every
call DataParallel scatters the frames over the GPUs and broadcasts all of the net's parameters to every replica; this
package never reads those copies (each replica runs on the net's handle for its GPU, which holds the weights already).
With one GPU DataParallel calls the module directly.

yolact_base (eval.py's default model) with deterministic weights, seeded 720x1280 frames.  The configurations
alternate, one window of --steps steps each per round, each window ending in a synchronise of every GPU used; the
median over rounds of frames / s is printed as one JSON line per (GPUs, video_multiframe), after one line with every
GPU's name and power limit.

    python scripts/bench_data_parallel.py [--gpus N] [--steps 20] [--warmup 3] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import yolact_b200
from oracle.weights import deterministic_state_dict
from yolact_b200.augmentations import FastBaseTransform
from yolact_b200.config import CONFIGS


class CustomDataParallel(torch.nn.DataParallel):
    """eval.py:630-634: gathers the replicas' lists of dicts without moving them."""
    def gather(self, outputs, output_device):
        return sum(outputs, [])


def gpu_info():
    """[(name, power limit)] of every visible GPU, from nvidia-smi (or torch, without a power limit)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return [tuple(s.strip() for s in line.split(",")) for line in q if line.strip()]
    except Exception:
        return [(torch.cuda.get_device_name(i), "unknown") for i in range(torch.cuda.device_count())]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=0, help="largest GPU count (default: every visible GPU)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--h", type=int, default=720)
    ap.add_argument("--w", type=int, default=1280)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_data_parallel.py measures on CUDA GPUs; none is visible")
    N = args.gpus or torch.cuda.device_count()
    if N > torch.cuda.device_count():
        raise SystemExit("--gpus %d: only %d GPUs are visible" % (N, torch.cuda.device_count()))
    print(json.dumps({"gpus": [{"name": n, "power_limit": p} for n, p in gpu_info()[:N]]}), flush=True)

    cfg = CONFIGS["yolact_base_config"].copy()
    yolact_b200.cfg.replace(cfg.copy())
    net = yolact_b200.Yolact(cfg, precision="f16x3")
    net.detect.use_fast_nms = True
    net.load_state_dict(deterministic_state_dict(net.state_dict(), 0))
    net.eval().cuda()

    g = torch.Generator().manual_seed(0)
    video = torch.randint(0, 256, (2 * N, args.h, args.w, 3), generator=g, dtype=torch.uint8)
    runs = []
    for n in range(1, N + 1):
        ids = list(range(n))
        dp = CustomDataParallel(net, device_ids=ids)
        transform = torch.nn.DataParallel(FastBaseTransform(cfg), device_ids=ids)
        for mf in sorted({1, N, 2 * N}):
            frames = [f.cuda().float() for f in video[:mf]]
            runs.append({"n": n, "mf": mf, "dp": dp, "transform": transform, "frames": frames, "fps": []})

    def step(r):
        return r["dp"](r["transform"](torch.stack(r["frames"], 0)))

    def window(r, steps):
        for d in range(r["n"]):
            torch.cuda.synchronize(d)
        t0 = time.perf_counter()
        for _ in range(steps):
            out = step(r)
        for d in range(r["n"]):
            torch.cuda.synchronize(d)
        assert len(out) == r["mf"]
        return time.perf_counter() - t0

    with torch.no_grad():
        for r in runs:
            window(r, args.warmup)     # handles, plans for each shard size, allocator
        for _ in range(args.rounds):
            for r in runs:
                r["fps"].append(r["mf"] * args.steps / window(r, args.steps))
    for r in runs:
        print(json.dumps({"gpus_used": r["n"], "video_multiframe": r["mf"], "frame": [args.h, args.w],
                          "frames_per_s": round(statistics.median(r["fps"]), 2),
                          "frames_per_s_rounds": [round(v, 2) for v in r["fps"]]}), flush=True)


if __name__ == "__main__":
    main()
