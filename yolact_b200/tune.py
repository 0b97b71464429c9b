"""Writes a plan file for a config, precision and list of input shapes, ahead of the processes that will use it.

    python -m yolact_b200.tune --config yolact_base_config --precision f16x3 --sizes 550 --batch 1,8 -o plans.txt

Builds the network with deterministic random weights and runs one forward per (batch, size): plans depend on the
shapes only (the autotuner times candidates on buffers whose contents do not matter), so the file serves any weights
of that config.  Load it with Yolact.load_plans(path), or YB_PLANS=path for every handle a process creates.  A file
is refused by another build of the library, another GPU model or SM count, another precision, or other YB_SK /
YB_CHAIN settings (include/yolact_b200.h, plan files).
"""
import argparse
import sys
import time


def _sizes(text):
    out = []
    for s in text.split(","):
        h, _, w = s.lower().partition("x")
        out.append((int(h), int(w or h)))
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m yolact_b200.tune", description=__doc__.split("\n\n")[0])
    ap.add_argument("--config", default="yolact_base_config")
    ap.add_argument("--precision", default="f16x3", choices=["f32", "f16tc", "f16x3"])
    ap.add_argument("--sizes", default="550", help="network input sizes: 550 or HxW, comma separated")
    ap.add_argument("--batch", default="1", help="batch sizes, comma separated")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--load", default=None, help="start from this plan file (its shapes are not timed again)")
    ap.add_argument("-o", "--output", required=True)
    a = ap.parse_args(argv)

    import torch
    from .config import CONFIGS, set_cfg
    from .yolact import Yolact

    name = a.config if a.config.endswith("_config") else a.config + "_config"
    if name not in CONFIGS:
        ap.error("unknown config %r (have: %s)" % (a.config, ", ".join(sorted(CONFIGS))))
    cfg = set_cfg(name).copy()
    dev = torch.device("cuda", a.device)
    torch.cuda.set_device(dev)
    torch.manual_seed(0)   # the parameters' own initialisers: deterministic random weights
    net = Yolact(cfg, precision=a.precision)
    net.train()
    if a.load:
        net.load_plans(a.load)
    for B in [int(b) for b in a.batch.split(",")]:
        for H, W in _sizes(a.sizes):
            t0 = time.perf_counter()
            net.forward_conv_only(torch.zeros(B, 3, H, W, device=dev))
            torch.cuda.synchronize(dev)
            timed, loaded = net.plan_stats(dev)
            print("B=%d %dx%d: %.1f s (decisions timed so far %d, taken from a file %d)"
                  % (B, H, W, time.perf_counter() - t0, timed, loaded), flush=True)
    net.save_plans(a.output, dev)
    print("wrote", a.output)
    return 0


if __name__ == "__main__":
    sys.exit(main())
