"""from_reference_cfg(): snapshotting the REAL reference cfg gives our named configs.  The raw fields of the reference's
own cfg objects that the converter reads are stored in tests/golden/reference_cfg.json (oracle/gen_golden.py `cfg`);
the test rebuilds duck-typed cfg objects from them and runs the converter."""
import copy
import json
import os
from types import SimpleNamespace

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load_reference_cfgs():
    return json.load(open(os.path.join(ROOT, "tests", "golden", "reference_cfg.json")))


def as_reference_cfg(raw):
    """A duck-typed reference cfg: attributes as in data/config.py, backbone.type a class of the stored name."""
    raw = copy.deepcopy(raw)
    bb = raw.pop("backbone")
    bb["type"] = type(bb["type"], (), {})
    bb["transform"] = SimpleNamespace(**bb["transform"])
    raw["fpn"] = SimpleNamespace(**raw["fpn"])
    return SimpleNamespace(backbone=SimpleNamespace(**bb), **raw)


def test_snapshot_matches_named_configs():
    from yolact_b200.config import CONFIGS, from_reference_cfg
    ref = load_reference_cfgs()
    assert sorted(ref) == sorted(CONFIGS)
    for name, mine in CONFIGS.items():
        snap = from_reference_cfg(as_reference_cfg(ref[name]))
        for key in ("backbone", "backbone_layers", "dcn_layers", "dcn_interval", "selected_layers", "max_size",
                    "pred_aspect_ratios", "use_square_anchors", "num_classes", "fpn_features", "use_maskiou",
                    "rescore_mask", "rescore_bbox", "nms_top_k", "nms_conf_thresh", "nms_thresh",
                    "max_num_detections", "normalize", "to_float"):
            assert getattr(snap, key) == getattr(mine, key), (name, key)
        for a, b in zip(snap.pred_scales, mine.pred_scales):
            assert [float(x) for x in a] == [float(x) for x in b], name


@pytest.mark.parametrize("switch, value", [("use_yolo_regressors", True), ("mask_proto_bias", True),
                                           ("share_prediction_module", False)])
def test_snapshot_rejects_unimplemented_switches(switch, value):
    from yolact_b200.config import from_reference_cfg
    raw = load_reference_cfgs()["yolact_base_config"]
    raw[switch] = value
    with pytest.raises(ValueError, match=switch):
        from_reference_cfg(as_reference_cfg(raw))


def test_snapshot_rejects_unknown_backbone():
    from yolact_b200.config import from_reference_cfg
    raw = load_reference_cfgs()["yolact_base_config"]
    raw["backbone"]["type"] = "VGGBackbone"
    with pytest.raises(ValueError, match="unsupported backbone"):
        from_reference_cfg(as_reference_cfg(raw))
