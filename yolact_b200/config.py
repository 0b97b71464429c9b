"""Configuration snapshot for the inference path.

The reference keeps a global mutable `cfg` (data/config.py:810) that the model both reads and writes
(yolact.py:425,445,567-568).  The H100 path takes an immutable snapshot of the ~30 keys it needs
(SURVEY.md Appendix C) at construction -- either from one of the named configs below or from any
object that quacks like the reference's `cfg` (`from_reference_cfg`).

Values mirror data/config.py: yolact_base_config (:656-704), yolact_im700_config (:715-723),
yolact_darknet53_config (:725-737), yolact_resnet50_config (:739-751), yolact_plus_base_config
(:772-792), yolact_plus_resnet50_config (:794-806), coco_base_config NMS keys (:424,450-454).
"""
import copy

# ImageNet statistics used by BaseTransform / FastBaseTransform (data/config.py:28-29), BGR order
MEANS = (103.94, 116.78, 123.68)
STD = (57.38, 57.12, 58.4)
# Display palette of prep_display (data/config.py:6-24), RGB
COLORS = ((244, 67, 54), (233, 30, 99), (156, 39, 176), (103, 58, 183), (63, 81, 181), (33, 150, 243), (3, 169, 244),
          (0, 188, 212), (0, 150, 136), (76, 175, 80), (139, 195, 74), (205, 220, 57), (255, 235, 59), (255, 193, 7),
          (255, 152, 0), (255, 87, 34), (121, 85, 72), (158, 158, 158), (96, 125, 139))


class Config(object):
    """Attribute dictionary with copy/replace, like the reference's Config (data/config.py:61-100)."""

    def __init__(self, d):
        for k, v in d.items():
            setattr(self, k, v)

    def copy(self, new=None):
        c = Config(copy.deepcopy(vars(self)))
        for k, v in (new or {}).items():
            setattr(c, k, v)
        return c

    def replace(self, other):
        if isinstance(other, Config):
            other = vars(other)
        for k, v in other.items():
            setattr(self, k, v)

    def __repr__(self):
        return "Config(%r)" % (vars(self),)


_PLUS_SCALES = [[float(s) * 2 ** (j / 3.0) for j in range(3)] for s in (24, 48, 96, 192, 384)]

_base = Config(dict(
    name="yolact_base",
    backbone="resnet", backbone_layers=[3, 4, 23, 3], dcn_layers=[0, 0, 0, 0], dcn_interval=1,
    selected_layers=[1, 2, 3],
    max_size=550,
    pred_scales=[[24], [48], [96], [192], [384]],
    pred_aspect_ratios=[1, 0.5, 2],
    use_square_anchors=True,
    num_classes=81, mask_dim=32, fpn_features=256,
    use_maskiou=False, rescore_mask=False, rescore_bbox=False,
    nms_top_k=200, nms_conf_thresh=0.05, nms_thresh=0.5, max_num_detections=100,
    eval_mask_branch=True, mask_proto_debug=False,
    normalize=True, to_float=False, subtract_means=False, channel_order="RGB",   # backbone.transform (config.py:181-202)
    preserve_aspect_ratio=False,        # config.py:655 (FastBaseTransform / Resize)
))

CONFIGS = {
    "yolact_base_config": _base,
    "yolact_resnet50_config": _base.copy(dict(name="yolact_resnet50", backbone_layers=[3, 4, 6, 3])),
    "yolact_im700_config": _base.copy(dict(
        name="yolact_im700", max_size=700,
        pred_scales=[[int(x[0] / 550.0 * 700)] for x in _base.pred_scales])),  # config.py:721
    "yolact_darknet53_config": _base.copy(dict(
        name="yolact_darknet53", backbone="darknet", backbone_layers=[1, 2, 8, 8, 4], selected_layers=[2, 3, 4],
        normalize=False, to_float=True)),
    "yolact_plus_base_config": _base.copy(dict(
        name="yolact_plus_base", dcn_layers=[0, 4, 23, 3], dcn_interval=3, pred_scales=_PLUS_SCALES,
        use_square_anchors=False, use_maskiou=True, rescore_mask=True, rescore_bbox=False)),
    "yolact_plus_resnet50_config": _base.copy(dict(
        name="yolact_plus_resnet50", backbone_layers=[3, 4, 6, 3], dcn_layers=[0, 4, 6, 3], dcn_interval=1,
        pred_scales=_PLUS_SCALES, use_square_anchors=False, use_maskiou=True, rescore_mask=True,
        rescore_bbox=False)),
}

# The package-level mutable config, like the reference's `cfg` global (data/config.py:810-821).
cfg = _base.copy()


def set_cfg(name):
    """set_cfg('yolact_base_config') -- same call the reference's eval.py makes (data/config.py:812-821)."""
    if not name.endswith("_config"):
        name = name + "_config"
    if name not in CONFIGS:
        raise KeyError("unknown config %r (have: %s)" % (name, ", ".join(sorted(CONFIGS))))
    cfg.replace(CONFIGS[name].copy())
    return cfg


def from_reference_cfg(rcfg):
    """Snapshot a reference-style cfg object (duck-typed) into this package's Config.

    Asserts the combination of switches the H100 path implements (every published config satisfies
    it); anything else must keep using the reference graph.
    """
    b = rcfg.backbone
    tname = getattr(b.type, "__name__", str(b.type))
    unsupported = []
    for key, want in (("use_prediction_module", False), ("use_yolo_regressors", False),
                      ("use_mask_scoring", False), ("use_instance_coeff", False),
                      ("use_focal_loss", False), ("use_objectness_score", False),
                      ("mask_proto_use_grid", False), ("mask_proto_coeff_gate", False),
                      ("mask_proto_prototypes_as_features", False),
                      ("mask_proto_split_prototypes_by_head", False), ("mask_proto_bias", False),
                      ("share_prediction_module", True)):
        if getattr(rcfg, key, want) != want:
            unsupported.append(key)
    if unsupported:
        raise ValueError("yolact_b200 does not implement cfg switches: %s" % ", ".join(unsupported))
    if "ResNet" in tname:
        backbone = "resnet"
        layers = list(b.args[0])
        dcn_layers = list(b.args[1]) if len(b.args) > 1 else [0, 0, 0, 0]
        dcn_interval = b.args[2] if len(b.args) > 2 else 1
    elif "DarkNet" in tname:
        backbone, layers, dcn_layers, dcn_interval = "darknet", list(b.args[0]), [0, 0, 0, 0], 1
    else:
        raise ValueError("yolact_b200: unsupported backbone %s" % tname)
    ars = b.pred_aspect_ratios[0][0]
    return Config(dict(
        name=getattr(rcfg, "name", "custom"),
        backbone=backbone, backbone_layers=layers, dcn_layers=dcn_layers, dcn_interval=dcn_interval,
        selected_layers=list(b.selected_layers), max_size=rcfg.max_size,
        pred_scales=[list(s) for s in b.pred_scales], pred_aspect_ratios=list(ars),
        use_square_anchors=bool(b.use_square_anchors),
        num_classes=rcfg.num_classes, mask_dim=getattr(rcfg, "mask_dim", 32) or 32,
        fpn_features=rcfg.fpn.num_features,
        use_maskiou=bool(getattr(rcfg, "use_maskiou", False)),
        rescore_mask=bool(getattr(rcfg, "rescore_mask", False)),
        rescore_bbox=bool(getattr(rcfg, "rescore_bbox", False)),
        nms_top_k=rcfg.nms_top_k, nms_conf_thresh=rcfg.nms_conf_thresh, nms_thresh=rcfg.nms_thresh,
        max_num_detections=rcfg.max_num_detections,
        eval_mask_branch=bool(getattr(rcfg, "eval_mask_branch", True)),
        mask_proto_debug=bool(getattr(rcfg, "mask_proto_debug", False)),
        normalize=bool(b.transform.normalize), to_float=bool(b.transform.to_float),
        subtract_means=bool(getattr(b.transform, "subtract_means", False)),
        channel_order=str(getattr(b.transform, "channel_order", "RGB")),
        preserve_aspect_ratio=bool(getattr(rcfg, "preserve_aspect_ratio", False)),
    ))
