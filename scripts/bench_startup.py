"""Start-up cost of a new input shape, with and without a plan file (yolact_base at 550^2, f16x3 unless --precision).

For each batch size, fresh processes (CUDA context and library already up, weights pushed) time with a host clock and
a device synchronise:
  first      the first net(x) in eval mode: executor construction (buffers, plans, chains), the forward and Detect;
  second     the next net(x), for the steady state the first call is compared with;
  build      the first forward_conv_only(x) of a second, fresh handle in the same process: executor construction
             plus one conv stack, without Detect -- with no file the plan decisions are timed here, with the file they
             are read from it;
and report the plan decisions timed and taken from the file (Yolact.plan_stats).  The plan file comes from
`python -m yolact_b200.tune` for the same batch sizes.  "no file" and "file" children alternate, --rounds times.
Prints the GPU name, power limit and SM clocks, which belong with every number, and one JSON line per child.

    python scripts/bench_startup.py [--batch 1,8] [--rounds 2] [--precision f16x3] [--out startup.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return "GPU details unknown"


def child(a):
    import torch
    import yolact_b200
    from yolact_b200.config import CONFIGS

    cfg = CONFIGS["yolact_base_config"].copy()
    yolact_b200.cfg.replace(cfg.copy())
    dev = torch.device("cuda", 0)
    x = torch.randn(a.B, 3, 550, 550, generator=torch.Generator().manual_seed(5)).to(dev)

    def make():
        torch.manual_seed(0)
        net = yolact_b200.Yolact(cfg, precision=a.precision)
        net.eval()
        if a.plans:
            net.load_plans(a.plans)
        net.num_priors_for(550, 550, dev)   # creates the handle and pushes the weights, outside the timed window
        torch.cuda.synchronize()
        return net

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    net = make()
    first = timed(lambda: net(x))
    second = timed(lambda: net(x))
    timed_n, loaded_n = net.plan_stats(dev)
    del net
    torch.cuda.empty_cache()
    net2 = make()
    build = timed(lambda: net2.forward_conv_only(x))
    t2, l2 = net2.plan_stats(dev)
    print(json.dumps(dict(B=a.B, plans=bool(a.plans), first_ms=round(first, 1), second_ms=round(second, 2),
                          build_ms=round(build, 1), timed=timed_n, loaded=loaded_n, build_timed=t2, build_loaded=l2)),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", default="1,8")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--precision", default="f16x3")
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--B", type=int, default=1, help=argparse.SUPPRESS)
    ap.add_argument("--plans", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        return child(a)

    print("GPU:", gpu_info(), flush=True)
    env = dict(os.environ)
    env.pop("YB_PLANS", None)
    batches = [int(b) for b in a.batch.split(",")]
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        plans = os.path.join(tmp, "plans.txt")
        t0 = time.perf_counter()
        subprocess.run([sys.executable, "-m", "yolact_b200.tune", "--config", "yolact_base_config", "--precision",
                        a.precision, "--sizes", "550", "--batch", a.batch, "-o", plans], cwd=ROOT, env=env, check=True)
        print("tune: %.1f s for batch %s" % (time.perf_counter() - t0, a.batch), flush=True)
        for r in range(a.rounds):
            for B in batches:
                for p in (None, plans):
                    cmd = [sys.executable, os.path.abspath(__file__), "--child", "--B", str(B), "--precision",
                           a.precision] + (["--plans", p] if p else [])
                    out = subprocess.run(cmd, cwd=ROOT, env=env, check=True, capture_output=True, text=True).stdout
                    row = json.loads(out.strip().splitlines()[-1])
                    print(json.dumps(row), flush=True)
                    rows.append(row)
    print("\n%-3s %-8s %12s %12s %12s %8s %8s" % ("B", "plans", "first ms", "second ms", "build ms", "timed", "loaded"))
    for B in batches:
        for p in (False, True):
            sel = [r for r in rows if r["B"] == B and r["plans"] == p]
            med = lambda k: statistics.median(r[k] for r in sel)
            rng = lambda k: "%.0f-%.0f" % (min(r[k] for r in sel), max(r[k] for r in sel))
            print("%-3d %-8s %12.1f %12.2f %12.1f %8d %8d   (first %s, build %s)" % (
                B, "file" if p else "none", med("first_ms"), med("second_ms"), med("build_ms"), sel[0]["timed"],
                sel[0]["loaded"], rng("first_ms"), rng("build_ms")))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(gpu=gpu_info(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
