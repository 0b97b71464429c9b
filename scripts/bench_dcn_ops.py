"""Time the dcn_v2 drop-in's general forward ops on the GPU, one op call at a time (CUDA events around `iters` calls
after `warmup` calls, the window ended by a synchronise):

  dcn_v2_conv in f32 / f16tc / f16x3 against torchvision.ops.deform_conv2d (fp32, with offset groups and mask) on the
  same inputs, at example_dconv's shape (2 x 64 x 128^2, deformable_groups 2), C = 256 with 4 groups at 69^2 and a 5x5
  kernel; dcn_v2_pooling at example_dpooling's shape (2 x 32 x 64^2, 20 RoIs) and a detection-sized load (300 RoIs, 7x7
  bins, 256-dim output over a 2 x 256 x 64^2 map).

An op call is what a user of the module pays: dcn_v2_conv packs the weights on the host and converts the layouts on
every call (the network's DCN layers do neither).  Prints the GPU's name and power limit and one JSON line.

    python scripts/bench_dcn_ops.py [--iters 20] [--warmup 3] [--out results/bench_dcn_ops.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from yolact_b200 import _lib  # noqa: E402
from yolact_b200.dcn_v2 import dcn_v2_conv, dcn_v2_pooling  # noqa: E402

CONV = [  # name, B, C, Co, H, W, k, pad, dg
    ("example_dconv 2x64x128^2 dg2", 2, 64, 64, 128, 128, 3, 1, 2),
    ("C256 dg4 69^2", 2, 256, 256, 69, 69, 3, 1, 4),
    ("5x5 C128 dg2 64^2", 2, 128, 128, 64, 64, 5, 2, 2),
]
POOL = [  # name, N, output_dim, H, W, R, pooled, no_trans
    ("example_dpooling 2x32x64^2 R20", 2, 32, 64, 64, 20, 7, False),
    ("detection 2x256x64^2 R300", 2, 256, 64, 64, 300, 7, False),
]


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dcn_ops.py measures on the GPU; none is visible")
    from torchvision.ops import deform_conv2d
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    res = {"gpu": gpu_info(), "unit": "ms per op call", "conv": {}, "pool": {}}
    print("GPU:", res["gpu"])
    for name, B, C, Co, H, W, k, pad, dg in CONV:
        x = torch.randn(B, C, H, W, device=dev, generator=g)
        w = torch.randn(Co, C, k, k, device=dev, generator=g) * (2.0 / (C * k * k)) ** 0.5
        bias = torch.randn(Co, device=dev, generator=g) * 0.1
        off = torch.randn(B, 2 * dg * k * k, H, W, device=dev, generator=g) * 2
        msk = torch.sigmoid(torch.randn(B, dg * k * k, H, W, device=dev, generator=g))
        row = {"torchvision_f32": timed(lambda: deform_conv2d(x, off, w, bias, padding=pad, mask=msk), args.iters,
                                        args.warmup)}
        ref = deform_conv2d(x, off, w, bias, padding=pad, mask=msk)
        for prec in ("f32", "f16tc", "f16x3"):
            try:
                y = dcn_v2_conv(x, off, msk, w, bias, 1, pad, 1, dg, precision=prec)
            except _lib.YbError as e:
                row[prec] = "refused: " + str(e).split(": ", 2)[-1].split(" [")[0]
                continue
            row[prec] = timed(lambda: dcn_v2_conv(x, off, msk, w, bias, 1, pad, 1, dg, precision=prec), args.iters,
                              args.warmup)
            row[prec + "_max_abs_diff_vs_torchvision"] = float((y - ref).abs().max())
        res["conv"][name] = row
        print(name, json.dumps(row))
    for name, N, D, H, W, R, P, no_trans in POOL:
        x = torch.randn(N, D, H, W, device=dev, generator=g)
        xy = torch.rand(R, 2, device=dev, generator=g) * 4 * W
        wh = torch.rand(R, 2, device=dev, generator=g) * W
        bidx = torch.randint(N, (R, 1), device=dev, generator=g).float()
        rois = torch.cat((bidx, xy, xy + wh), dim=1)
        trans = torch.randn(R, 2, P, P, device=dev, generator=g)
        row = {"dcn_v2_pooling": timed(lambda: dcn_v2_pooling(x, rois, trans, 0.25, P, D, no_trans, 1, P, 4, 0.1),
                                       args.iters, args.warmup)}
        res["pool"][name] = row
        print(name, json.dumps(row))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
