"""ctypes binding of libyolact_b200.so (the C ABI in include/yolact_b200.h).

The product path has NO CPU fallback: if the shared library is missing or no H100 is visible the
calls below raise -- they never route to the oracle or to PyTorch ops.
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("YB_LIB") or os.path.join(_HERE, "libyolact_b200.so")


class YbConfig(ctypes.Structure):
    """Mirror of yb_config."""
    _fields_ = [
        ("backbone", c_int32),
        ("num_stages", c_int32),
        ("layers", c_int32 * 5),
        ("dcn_layers", c_int32 * 4),
        ("dcn_interval", c_int32),
        ("selected_layers", c_int32 * 3),
        ("max_size", c_int32),
        ("num_classes", c_int32),
        ("mask_dim", c_int32),
        ("fpn_features", c_int32),
        ("num_scales", c_int32),
        ("scales", (c_float * 4) * 5),
        ("num_ars", c_int32),
        ("ars", c_float * 4),
        ("use_square_anchors", c_int32),
        ("use_maskiou", c_int32),
        ("precision", c_int32),
        ("nms_top_k", c_int32),
        ("nms_conf_thresh", c_float),
        ("nms_thresh", c_float),
        ("max_num_detections", c_int32),
        ("scales_f64", (ctypes.c_double * 4) * 5),
        ("ars_f64", ctypes.c_double * 4),
    ]


class YbPostItem(ctypes.Structure):
    """Mirror of yb_post_item (one image of yb_postprocess_list)."""
    _fields_ = [
        ("proto", c_void_p),
        ("coef", c_void_p),
        ("box", c_void_p),
        ("masks", c_void_p),
        ("boxes_px", c_void_p),
        ("proto_masks", c_void_p),
        ("n", c_int32),
        ("out_h", c_int32),
        ("out_w", c_int32),
    ]


class YbEvalIouItem(ctypes.Structure):
    """Mirror of yb_eval_iou_item (one image of yb_eval_iou_list)."""
    _fields_ = [
        ("proto", c_void_p),
        ("coef", c_void_p),
        ("box", c_void_p),
        ("boxes_px", c_void_p),
        ("gt_bits", c_void_p),
        ("gt_boxes", c_void_p),
        ("box_iou", c_void_p),
        ("mask_iou", c_void_p),
        ("crowd_box_iou", c_void_p),
        ("crowd_mask_iou", c_void_p),
        ("n", c_int32),
        ("out_h", c_int32),
        ("out_w", c_int32),
        ("g_all", c_int32),
        ("num_crowd", c_int32),
    ]


class YbEvalMatchItem(ctypes.Structure):
    """Mirror of yb_eval_match_item (one image of yb_eval_match_list)."""
    _fields_ = [
        ("box_iou", c_void_p),
        ("mask_iou", c_void_p),
        ("crowd_box_iou", c_void_p),
        ("crowd_mask_iou", c_void_p),
        ("cls", c_void_p),
        ("box_score", c_void_p),
        ("mask_score", c_void_p),
        ("gt_cls", c_void_p),
        ("crowd_cls", c_void_p),
        ("rec_offset", c_int64),
        ("n", c_int32),
        ("g", c_int32),
        ("num_crowd", c_int32),
    ]


class YbRenderItem(ctypes.Structure):
    """Mirror of yb_render_item (one frame of yb_render_list)."""
    _fields_ = [
        ("frame", c_void_p),
        ("out", c_void_p),
        ("proto", c_void_p),
        ("coef", c_void_p),
        ("box", c_void_p),
        ("cls", c_void_p),
        ("score", c_void_p),
        ("det_score", c_void_p),
        ("sel_n", c_void_p),
        ("sel_cls", c_void_p),
        ("sel_score", c_void_p),
        ("sel_box", c_void_p),
        ("n", c_int32),
        ("h", c_int32),
        ("w", c_int32),
    ]


class YbRenderOpts(ctypes.Structure):
    """Mirror of yb_render_opts (yb_render_list_ex)."""
    _fields_ = [
        ("d_counts", c_void_p),
        ("fps_w", c_int32),
        ("fps_h", c_int32),
        ("draw_masks", c_int32),
    ]


class YbConvOpts(ctypes.Structure):
    """Mirror of yb_conv_opts (yb_conv2d_ex)."""
    _fields_ = [
        ("res_after_act", c_int32),
        ("y_f32", c_int32),
        ("cin_pad", c_int32),
        ("cout_pad", c_int32),
        ("y_pix_stride", c_int32),
        ("poison", c_int32),
        ("nseg", c_int32),
        ("seg_begin", c_int32 * 3),
        ("seg_end", c_int32 * 3),
        ("seg_act", c_int32 * 3),
        ("seg_pix_stride", c_int32 * 3),
        ("seg_batch_stride", c_int64 * 3),
        ("seg_y", c_void_p * 3),
    ]


class YbDcnParams(ctypes.Structure):
    """Mirror of yb_dcn_params (yb_dcn_forward_ex)."""
    _fields_ = [
        ("kernel_h", c_int32), ("kernel_w", c_int32),
        ("stride_h", c_int32), ("stride_w", c_int32),
        ("pad_h", c_int32), ("pad_w", c_int32),
        ("dilation_h", c_int32), ("dilation_w", c_int32),
        ("deformable_group", c_int32),
    ]


YB_BACKBONE_NONE, YB_BACKBONE_RESNET, YB_BACKBONE_DARKNET = -1, 0, 1
YB_PREC_F32, YB_PREC_F16TC, YB_PREC_F16X3 = 0, 1, 2
PRECISIONS = {"f32": YB_PREC_F32, "f16tc": YB_PREC_F16TC, "f16x3": YB_PREC_F16X3}
YB_MASK_F32, YB_MASK_U8, YB_MASK_BITS = 0, 1, 2
YB_NMS_FAST, YB_NMS_CROSS_CLASS, YB_NMS_TRADITIONAL = 0, 1, 2
YB_NMS_FLAG_SECOND_THRESHOLD = 0x100
YB_XFORM_NORMALIZE, YB_XFORM_SUBTRACT_MEANS, YB_XFORM_TO_FLOAT, YB_XFORM_NONE = 0, 1, 2, 3
YB_RESAMPLE_MAXPOOL, YB_RESAMPLE_BILINEAR = 0, 1

# name -> (restype, argtypes); kept in one table so tests can check that every symbol the header
# declares is exported by the library.
ABI_VERSION = 2   # include/yolact_b200.h YB_ABI_VERSION
SIGNATURES = {
    "yb_abi_version": (c_int, []),
    "yb_last_error": (c_char_p, []),
    "yb_device_count": (c_int, []),
    "yb_create": (c_int, [POINTER(YbConfig), c_int, POINTER(c_void_p)]),
    "yb_destroy": (c_int, [c_void_p]),
    "yb_load_weight": (c_int, [c_void_p, c_char_p, c_void_p, POINTER(c_int64), c_int]),
    "yb_finalize_weights": (c_int, [c_void_p]),
    "yb_num_priors": (c_int, [c_void_p, c_int, c_int, POINTER(c_int64), POINTER(c_int32)]),
    "yb_priors": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "yb_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "yb_proto_size": (c_int, [c_void_p, c_int, c_int, POINTER(c_int32), POINTER(c_int32)]),
    "yb_debug_feature": (c_int, [c_void_p, c_int, c_void_p, POINTER(c_int32), c_void_p]),
    "yb_softmax": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "yb_detect": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int64, c_int, c_int, c_int,
                          c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "yb_set_detect_params": (c_int, [c_void_p, c_int, c_float, c_float, c_int]),
    "yb_infer": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                         c_void_p, c_void_p, c_void_p, c_void_p]),
    "yb_infer_frames": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                POINTER(c_float), POINTER(c_float), c_int, c_int, c_void_p, c_void_p, c_void_p,
                                c_void_p, c_void_p, c_void_p, c_void_p]),
    "yb_infer_frame_list": (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_int32), c_int, c_int, c_int, c_int,
                                    POINTER(c_float), POINTER(c_float), c_int, c_int, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_void_p]),
    "yb_postprocess": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                               c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "yb_postprocess_batch": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                     c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "yb_postprocess_list": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "yb_coco_rle_list": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int64, c_void_p,
                                 c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "yb_maskiou": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "yb_fast_base_transform": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                       POINTER(c_float), POINTER(c_float), c_void_p, c_void_p]),
    "yb_pack_mask_bits": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int, c_void_p, c_void_p]),
    "yb_mask_iou": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int64, c_int, c_void_p, c_void_p]),
    "yb_box_iou": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "yb_mask_rle": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int64, c_void_p, c_void_p]),
    "yb_eval_match": (c_int, [c_void_p] + [c_void_p] * 7 + [c_int, c_void_p, c_int, c_void_p, c_int,
                                                              POINTER(ctypes.c_double), c_int, c_int] + [c_void_p] * 5),
    "yb_eval_iou_list": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "yb_eval_match_list": (c_int, [c_void_p, c_void_p, c_int, POINTER(ctypes.c_double), c_int, c_int] + [c_void_p] * 5),
    "yb_eval_ap_workspace": (c_int, [c_int64, c_int, c_int, POINTER(c_int64)]),
    "yb_eval_ap": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_int, c_int, c_void_p, c_int64, c_void_p,
                           c_void_p, c_void_p]),
    "yb_pack_detections": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                   c_void_p, c_void_p]),
    "yb_display_blend": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_float,
                                 c_void_p, c_void_p]),
    "yb_render_list": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_int,
                               c_float, c_void_p, c_int, c_void_p]),
    "yb_render_list_ex": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_int,
                                  c_float, c_void_p, c_int, POINTER(YbRenderOpts), c_void_p]),
    "yb_dcn_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 14 +
                       [c_void_p]),
    "yb_dcn_forward_ex": (c_int, [c_void_p] * 7 + [c_int] * 5 + [POINTER(YbDcnParams), c_void_p]),
    "yb_dcn_psroi_pool": (c_int, [c_void_p] * 6 + [c_int] * 7 + [c_float] + [c_int] * 5 + [c_float, c_void_p]),
    "yb_conv2d": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 12 +
                  [POINTER(c_float), c_void_p]),
    "yb_conv2d_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 11 +
                     [POINTER(YbConvOpts), c_void_p]),
    "yb_resample_ex": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 7 + [c_void_p]),
    "yb_launch_count": (c_int64, [c_void_p]),
    "yb_set_profiling": (c_int, [c_void_p, c_int]),
    "yb_last_forward_ms": (c_int, [c_void_p, POINTER(c_float), POINTER(c_float)]),
    "yb_last_forward_profile": (c_int, [c_void_p, c_char_p, c_int64]),
    "yb_debug_chain_deps": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_int32)]),
    "yb_set_graphs": (c_int, [c_void_p, c_int]),
    "yb_save_plans": (c_int, [c_void_p, c_char_p]),
    "yb_load_plans": (c_int, [c_void_p, c_char_p]),
    "yb_plan_stats": (c_int, [c_void_p, POINTER(c_int64), POINTER(c_int64)]),
    "yb_build_id": (c_char_p, []),
    "yb_check_plans": (c_int, [c_char_p, c_char_p]),
}

_lib = None


class YbError(RuntimeError):
    pass


def load():
    """Loads the shared library (building nothing: run `python -m yolact_b200.build` first)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise YbError(
            "yolact_b200: %s is missing. Build it with `python -m yolact_b200.build` "
            "(nvcc, sm_90a). There is no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.yb_abi_version() != ABI_VERSION:
        raise YbError("yolact_b200: ABI version mismatch")
    _lib = lib
    return lib


def check(status, what=""):
    if status != 0:
        msg = load().yb_last_error()
        raise YbError("%s failed (status %d): %s" % (what or "yolact_b200 call", status,
                                                     msg.decode() if msg else "?"))


def ptr(t):
    """data_ptr of a torch tensor (or None) as c_void_p."""
    if t is None:
        return c_void_p(0)
    return c_void_p(t.data_ptr())


def current_stream(device=None):
    import torch
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)
