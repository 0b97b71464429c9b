#!/usr/bin/env python
"""Full-size parity report: GPU path (a precision mode) vs the CPU oracle on the BASELINE configs.

    python scripts/parity_report.py --precisions f16tc,f16x3 --out parity.json

One row per (config, precision): raw head-tensor error (max |d| / max |ref|), class ids equal, keep-set
agreement, max |dbox|, max |dscore|, flipped mask pixels, as a markdown table on stdout.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [  # (config, size, batch, out_hw): BASELINE.json configs 2-5 shapes (batch bounded by the CPU oracle's time)
    ("yolact_base_config", 550, 2, (550, 550)),
    ("yolact_base_config", 550, 1, (480, 640)),          # eval.py:266 postprocess target of a 640x480 frame
    ("yolact_plus_resnet50_config", 550, 2, (550, 550)),
    ("yolact_im700_config", 700, 1, (700, 700)),
    ("yolact_plus_base_config", 550, 1, (550, 550)),
    ("yolact_resnet50_config", 550, 1, (550, 550)),
    ("yolact_darknet53_config", 416, 1, (416, 416)),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precisions", default="f16tc")
    ap.add_argument("--cases", default="")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    from tests.parity_utils import measure
    from yolact_b200.config import CONFIGS
    rows = []
    sel = [int(i) for i in a.cases.split(",")] if a.cases else range(len(CASES))
    print("| config | size | B | out | mode | raw loc | raw conf | raw coef | raw proto | cls ids equal (strict / mod ties<2e-5) | keep-set | max dbox | max dscore | mask flips |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|---|---|")
    for ci in sel:
        name, size, batch, out_hw = CASES[ci]
        cfg = CONFIGS[name].copy()
        for prec in a.precisions.split(","):
            t0 = time.time()
            r = measure(cfg, prec, batch, size, out_hw)
            r["seconds"] = time.time() - t0
            rows.append(r)
            f = lambda v: "-" if v is None else ("%.2e" % v)
            print("| %s | %d | %d | %dx%d | %s | %s | %s | %s | %s | %s (%d/%d) | %s | %s | %s | %s |" % (
                cfg.name, size, batch, out_hw[0], out_hw[1], prec, f(r["raw_loc"]), f(r["raw_conf"]), f(r["raw_mask"]),
                f(r["raw_proto"]), "%s / %s" % (r["class_ids_equal_strict"], r["class_ids_equal"]), r["class_ids_equal_images"], r["images"],
                f(r["keep_set_agreement_min"]), f(r["max_abs_dbox"]), f(r["max_abs_dscore"]),
                f(r["mask_pixel_mismatch_max"])), flush=True)
    if a.out:
        json.dump(rows, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
