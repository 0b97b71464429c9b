"""Full-size end-to-end parity of the BENCHED precision mode (f16x3, split-precision tensor-core) on the BASELINE.json
configs: `net(x)` in eval mode + `postprocess()` on the GPU against the CPU oracle (pinned to the reference by the
goldens), with north_star's bar: class ids identical, boxes / scores within 1e-3, < 1e-3 mismatching mask pixels.
The single-pass fp16 mode is measured by the same code and only bounded loosely (it is the labelled fast mode)."""
import pytest

from tests.helpers import cfg_for
from tests.parity_utils import measure

pytestmark = pytest.mark.gpu

# (config, size, batch, postprocess target (h, w)) -- batch bounded by the CPU oracle's time (DCN in numpy)
CASES = [
    ("yolact_base_config", 550, 2, (550, 550)),            # BASELINE configs[1]
    ("yolact_base_config", 550, 1, (480, 640)),            # eval.py:266: masks at the ORIGINAL 640x480 frame size
    ("yolact_plus_resnet50_config", 550, 1, (550, 550)),   # configs[2]
    ("yolact_im700_config", 700, 1, (700, 700)),           # configs[3]
    ("yolact_plus_base_config", 550, 1, (550, 550)),       # configs[4]
    ("yolact_resnet50_config", 550, 1, (550, 550)),        # configs[0]
    ("yolact_darknet53_config", 416, 1, (416, 416)),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "%s@%d->%dx%d" % (c[0].replace("_config", ""), c[1], c[3][0], c[3][1]))
def test_benched_mode_meets_north_star_tolerance(case):
    name, size, batch, out_hw = case
    r = measure(cfg_for(name), "f16x3", batch, size, out_hw)
    print({k: v for k, v in r.items() if k != "counts_gpu_ref"})
    assert r["priors_equal"]
    for k in ("raw_loc", "raw_conf", "raw_mask", "raw_proto"):
        assert r[k] < 2e-4, (k, r[k])
    assert r["class_ids_equal"], r["counts_gpu_ref"]                  # bit-exact class indices, same order
    assert r["keep_set_agreement_min"] == 1.0
    assert r["max_abs_dbox"] < 1e-3 and r["max_abs_dscore"] < 1e-3   # north_star: 1e-3 on boxes
    assert r["max_abs_dbox_px"] <= 1                                 # .long() of x*w at fp32 rounding noise
    assert r["mask_pixel_mismatch_max"] < 1e-3                       # north_star: 1e-3 on masks
    if r["max_abs_dscore_maskiou"] is not None:
        assert r["max_abs_dscore_maskiou"] < 1e-3


def test_fast_mode_is_bounded():
    r = measure(cfg_for("yolact_base_config"), "f16tc", 1, 550)
    print({k: v for k, v in r.items() if k != "counts_gpu_ref"})
    for k in ("raw_loc", "raw_conf", "raw_proto"):
        assert r[k] < 5e-3, (k, r[k])
    assert r["raw_mask"] < 4e-2
    assert r["keep_set_agreement_min"] >= 0.85
