/*
 * yolact_b200.h -- C ABI of the H100-native YOLACT inference path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  Every entry point takes
 * plain pointers / sizes / a cudaStream_t passed as void*; there are no torch
 * types in any signature.  Pointers named `d_*` are DEVICE pointers owned by
 * the caller; `h_*` are HOST pointers.  The library owns only weights, plans
 * and workspaces (all inside the opaque handle).
 *
 * Every function returns 0 on success or a negative yb_status; the message of
 * the last failure on the calling thread is available from yb_last_error().
 * (The reference reports CUDA launch errors with printf only,
 * external/DCNv2/src/cuda/dcn_v2_im2col_cuda.cu:346-350; we surface them.)
 *
 * Reference interfaces replaced (all paths relative to the reference root):
 *   yb_create / yb_load_weight / yb_finalize_weights
 *        <- Yolact.__init__ (yolact.py:399-471), Yolact.load_weights (yolact.py:477-490)
 *   yb_priors          <- PredictionModule.make_priors (yolact.py:214-263)
 *   yb_forward         <- Yolact.forward up to pred_outs (yolact.py:564-647), i.e.
 *                         ResNetBackbone.forward (backbone.py:126-139) / DarkNetBackbone.forward
 *                         (backbone.py:299-309), FPN.forward (yolact.py:311-361), proto_net
 *                         (utils/functions.py:163-213, yolact.py:588-599),
 *                         PredictionModule.forward (yolact.py:133-212)
 *   yb_softmax         <- F.softmax(conf, -1) (yolact.py:674)
 *   yb_detect          <- Detect.__call__/detect/fast_nms/cc_fast_nms (layers/functions/detection.py:32-180)
 *                         with decode (layers/box_utils.py:267-312) and jaccard (box_utils.py:54-80)
 *   yb_postprocess     <- postprocess lincomb path (layers/output_utils.py:15-99), crop and
 *                         sanitize_coordinates (layers/box_utils.py:327-373), F.interpolate bilinear
 *   yb_postprocess_list <- the same, called once per image of a batch of differently sized images (evalimages over a
 *                         folder, eval.py:612-625)
 *   yb_coco_rle_list   <- postprocess + pycocotools.mask.encode + rleToString in prep_metrics' --output_coco_json path
 *                         (eval.py:320-330, :414-429), for a list of images, without materialising masks
 *   yb_maskiou         <- FastMaskIoUNet.forward (yolact.py:363-375) + gather (output_utils.py:79-83)
 *   yb_fast_base_transform <- FastBaseTransform.forward (utils/augmentations.py:616-658)
 *   yb_infer_frames    <- FastBaseTransform()(frames) followed by Yolact.forward in eval mode, as evalimage /
 *                         evalvideo call them (eval.py:597-598, :695-704)
 *   yb_infer_frame_list <- the same for a batch of differently sized frames (evalimages over a folder, eval.py:612-625)
 *   yb_mask_iou / yb_box_iou <- mask_iou / jaccard (layers/box_utils.py:98-113, :54-79) as used by
 *                         eval.py:435-445 (_mask_iou, _bbox_iou)
 *   yb_mask_rle        <- pycocotools.mask.encode in Detections.add_mask (eval.py:320-330)
 *   yb_eval_match      <- prep_metrics' score orders and detection-to-ground-truth matching loop (eval.py:431-509)
 *   yb_eval_ap         <- APDataObject.get_ap / is_empty (eval.py:513-581) for every (type, threshold, class) cell
 *   yb_display_blend   <- the GPU mask blend of prep_display (eval.py:186-209,226)
 *   yb_render_list     <- the GPU part of prep_display with undo_transform=False (eval.py:147-226): postprocess with
 *                         rescore_bbox, top-k selection, score cut, palette, mask blend and .byte(), for a list of
 *                         frames, without materialising masks
 *   yb_render_list_ex  <- the same with device row counts (yb_infer_frames' padded outputs, no host sync), the
 *                         --display_fps box (eval.py:211-219) and --display_masks=False
 *   yb_dcn_forward     <- dcn_v2_forward (external/DCNv2/src/dcn_v2.h:9-39,
 *                         src/cuda/dcn_v2_cuda.cu:42-172, src/cuda/dcn_v2_im2col_cuda.cu:125-195)
 *   yb_dcn_forward_ex  <- the same for any kernel size, anisotropic geometry and deformable groups
 *   yb_dcn_psroi_pool  <- dcn_v2_psroi_pooling_forward (src/cuda/dcn_v2_psroi_pooling_cuda.cu:59-146)
 *   yb_conv2d          <- nn.Conv2d + folded BatchNorm2d + activation (+ residual), op-level test hook
 *   yb_conv2d_ex       <- the same with the network's other epilogues (residual after the activation, fp32 output,
 *                         zero-padded channels, the fused prediction head) and the tensor-core stem, op-level test hook
 *   yb_resample_ex     <- nn.MaxPool2d(3, 2, 1) (backbone.py:80) and F.interpolate bilinear (+ lateral, + ReLU) of the
 *                         FPN (yolact.py:332) and protonet (utils/functions.py:194), op-level test hook
 */
#ifndef YOLACT_B200_H_
#define YOLACT_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YB_ABI_VERSION 2   /* 2: yb_config gained scales_f64 / ars_f64, YB_PREC_F16X3, yb_set_detect_params */

#if defined(__GNUC__)
#define YB_API __attribute__((visibility("default")))
#else
#define YB_API
#endif

typedef enum {
  YB_OK = 0,
  YB_ERR_INVALID = -1,      /* bad argument / unsupported configuration */
  YB_ERR_CUDA = -2,         /* a CUDA runtime / driver call failed        */
  YB_ERR_STATE = -3,        /* call order violated (e.g. forward before finalize) */
  YB_ERR_MISSING_WEIGHT = -4,
  YB_ERR_NO_DEVICE = -5
} yb_status;

typedef enum { YB_BACKBONE_NONE = -1, YB_BACKBONE_RESNET = 0, YB_BACKBONE_DARKNET = 1 } yb_backbone;

/* Arithmetic mode of the convolution stack.
 *   YB_PREC_F32  : fp32 activations, fp32 FMA on CUDA cores (reference-order arithmetic, slow; second opinion)
 *   YB_PREC_F16TC: fp16 activations/weights, fp32 accumulation on the tensor cores (wgmma): one MMA pass, 11-bit
 *                  operands -- the fast mode; head tensors within ~2e-3 of range of the fp32 reference
 *   YB_PREC_F16X3: split precision on the tensor cores (the default of the Python API): every activation and weight is
 *                  an fp16 pair hi + lo (22 significand bits), each k-block issues hi*hi + lo*hi + hi*lo into fp32
 *                  register accumulators -- fp32-equivalent results (1e-3 on boxes/masks, identical class ids
 *                  against the fp32 reference) at three MMA passes and twice the operand bytes */
typedef enum { YB_PREC_F32 = 0, YB_PREC_F16TC = 1, YB_PREC_F16X3 = 2 } yb_precision;

/* Detect's NMS variant (the `cross_class` argument of yb_detect / yb_infer):
 *   YB_NMS_FAST        : fast_nms          (detection.py:137-180; eval.py default)
 *   YB_NMS_CROSS_CLASS : cc_fast_nms       (detection.py:111-135; --cross_class_nms)
 *   YB_NMS_TRADITIONAL : traditional_nms   (detection.py:182-228 + utils/cython_nms.pyx; --fast_nms=False) */
typedef enum { YB_NMS_FAST = 0, YB_NMS_CROSS_CLASS = 1, YB_NMS_TRADITIONAL = 2 } yb_nms_mode;
/* OR-ed into the nms mode: fast_nms(second_threshold=True), i.e. a kept detection must also have its OWN class score
 * above conf_thresh (detection.py:155-161; the reference leaves it off, "+0.2 mAP for 34 -> 33 fps"). YB_NMS_FAST only. */
#define YB_NMS_FLAG_SECOND_THRESHOLD 0x100

/* cfg.backbone.transform of FastBaseTransform (utils/augmentations.py:645-650) */
typedef enum {
  YB_XFORM_NORMALIZE = 0,       /* (x - mean) / std   (all published configs except darknet53) */
  YB_XFORM_SUBTRACT_MEANS = 1,  /* x - mean                                                     */
  YB_XFORM_TO_FLOAT = 2,        /* x / 255            (yolact_darknet53)                        */
  YB_XFORM_NONE = 3
} yb_transform_mode;

/* Output formats of yb_postprocess masks. */
typedef enum {
  YB_MASK_F32 = 0,   /* float 0/1, [n, h, w]           -- exactly what the reference returns   */
  YB_MASK_U8 = 1,    /* uint8 0/1, [n, h, w]                                                   */
  YB_MASK_BITS = 2   /* 1 bit / pixel, little-endian in uint32 words, row pitch = ceil(w/32) words */
} yb_mask_format;

/* Immutable snapshot of the cfg keys the inference path reads (SURVEY.md Appendix C).
 * All six published configs differ only in these fields. */
typedef struct {
  int32_t backbone;            /* yb_backbone */
  int32_t num_stages;          /* 4 for ResNet, 5 for Darknet                              */
  int32_t layers[5];           /* blocks per stage: {3,4,23,3} R101, {3,4,6,3} R50, {1,2,8,8,4} D53 */
  int32_t dcn_layers[4];       /* ResNetBackbone dcn_layers (backbone.py:62)               */
  int32_t dcn_interval;        /* >= 1                                                      */
  int32_t selected_layers[3];  /* cfg.backbone.selected_layers                              */
  int32_t max_size;            /* cfg.max_size (550 / 700); anchors use pixel scales        */
  int32_t num_classes;         /* 81 (incl. background)                                     */
  int32_t mask_dim;            /* 32                                                        */
  int32_t fpn_features;        /* 256                                                       */
  int32_t num_scales;          /* scales per level: 1, or 3 for YOLACT++                    */
  float   scales[5][4];        /* cfg.backbone.pred_scales                                  */
  int32_t num_ars;             /* 3                                                         */
  float   ars[4];              /* {1, 0.5, 2}                                               */
  int32_t use_square_anchors;  /* config.py:675 bug-compat                                  */
  int32_t use_maskiou;         /* YOLACT++ FastMaskIoUNet                                   */
  int32_t precision;           /* yb_precision                                              */
  int32_t nms_top_k;           /* 200  */
  float   nms_conf_thresh;     /* 0.05 */
  float   nms_thresh;          /* 0.5  */
  int32_t max_num_detections;  /* 100  */
  /* The reference evaluates the anchors in Python doubles from the un-rounded config values and rounds to fp32 once at
   * the end (yolact.py:224-246); YOLACT++'s scales 24 * 2^(j/3) are not fp32 numbers.  Non-zero entries here take
   * precedence over scales[][] / ars[] so that the priors are bit-identical to the reference's for every config. */
  double  scales_f64[5][4];
  double  ars_f64[4];
} yb_config;

typedef struct yb_handle yb_handle;

/* ---- lifecycle ----------------------------------------------------------------------------- */
YB_API int yb_abi_version(void);
YB_API const char* yb_last_error(void);
/* Number of CUDA devices visible; negative status if the runtime cannot initialise. */
YB_API int yb_device_count(void);
/* cfg->backbone == YB_BACKBONE_NONE creates an "ops only" handle (detect / postprocess / dcn). */
YB_API int yb_create(const yb_config* cfg, int device, yb_handle** out);
YB_API int yb_destroy(yb_handle* h);

/* ---- weights (reference state_dict names, Appendix B) ---------------------------------------- */
/* h_data: host fp32, contiguous, `ndim` dims in `shape` (PyTorch OIHW for conv weights). Unknown
 * names (semantic_seg_conv.*, num_batches_tracked) are accepted and ignored, like load_weights. */
YB_API int yb_load_weight(yb_handle* h, const char* name, const float* h_data, const int64_t* shape, int ndim);
/* Folds BatchNorm (eps 1e-5) into conv weight/bias, repacks for the kernels, uploads. */
YB_API int yb_finalize_weights(yb_handle* h);

/* ---- priors ---------------------------------------------------------------------------------- */
/* Number of priors for an (img_h,img_w) input; also returns the 5 feature-map sizes (may be NULL). */
YB_API int yb_num_priors(yb_handle* h, int img_h, int img_w, int64_t* num_priors, int32_t* level_hw /*[5][2]*/);
/* Writes [P,4] (cx,cy,w,h) fp32 priors to device memory. */
YB_API int yb_priors(yb_handle* h, int img_h, int img_w, float* d_priors, void* stream);

/* ---- network --------------------------------------------------------------------------------- */
/* x: NCHW fp32 [B,3,H,W] (already normalised, like Yolact.forward's input).
 * Outputs (fp32, caller allocated): loc [B,P,4], conf [B,P,num_classes] RAW LOGITS,
 * coef [B,P,mask_dim] (tanh applied), proto [B,ph,pw,mask_dim] NHWC (relu applied).
 * Any output pointer may be NULL to skip the copy-out of that tensor. */
YB_API int yb_forward(yb_handle* h, const float* d_x, int B, int H, int W,
               float* d_loc, float* d_conf, float* d_coef, float* d_proto, void* stream);
YB_API int yb_proto_size(yb_handle* h, int img_h, int img_w, int32_t* ph, int32_t* pw);
/* Returns backbone/FPN feature maps for tests: which = 0..3 backbone stage outputs C2..C5 (NHWC->NCHW fp32),
 * 4..8 = FPN P3..P7.  d_out must hold B*C*H*W floats; dims returned in chw[3]. */
YB_API int yb_debug_feature(yb_handle* h, int which, float* d_out, int32_t* chw, void* stream);

/* row-wise softmax over the last dim, rows x cols fp32 (in place allowed) */
YB_API int yb_softmax(yb_handle* h, const float* d_in, float* d_out, int64_t rows, int cols, void* stream);

/* ---- Detect ---------------------------------------------------------------------------------- */
/* conf_is_logits: 1 -> softmax is fused into candidate selection (conf untouched);
 *                 0 -> conf already softmaxed (what the reference Detect receives).
 * cross_class: a yb_nms_mode: 0 -> fast_nms (per class), 1 -> cc_fast_nms, 2 -> traditional_nms (greedy per-class
 * NMS on boxes scaled by cfg.max_size with the +1 pixel convention; needs max_num_detections <= nms_top_k).
 * Outputs per image, padded to max_out rows (max_out >= max_num_detections, or >= nms_top_k when
 * cross_class): box [B,max_out,4] relative x1y1x2y2, coef [B,max_out,mask_dim], cls int64
 * [B,max_out] in [0,num_classes-1), score [B,max_out] descending, count int32 [B] (0 == the
 * reference's `None`). */
YB_API int yb_detect(yb_handle* h, const float* d_loc, const float* d_conf, const float* d_coef,
              const float* d_priors, int B, int64_t P, int conf_is_logits, int cross_class,
              int max_out, float* d_box, float* d_coef_out, int64_t* d_cls, float* d_score,
              int32_t* d_count, void* stream);

/* Detect's parameters (Detect.top_k / conf_thresh / nms_thresh and cfg.max_num_detections, detection.py:17-31) are taken
 * from yb_config at yb_create; the reference lets callers change the attributes of net.detect afterwards, this is the
 * C-side of that.  Changing them synchronises the device and drops the captured yb_infer graphs. */
YB_API int yb_set_detect_params(yb_handle* h, int top_k, float conf_thresh, float nms_thresh, int max_num_detections);

/* Fused eval-mode path: yb_forward + yb_detect on the library's internal head buffers (no copy-out
 * of loc/conf/coef).  This is Yolact.forward() in eval mode (yolact.py:649-676).  d_proto
 * [B,ph,pw,mask_dim] receives the prototypes (nullable).  Replayed as one CUDA graph. */
YB_API int yb_infer(yb_handle* h, const float* d_x, int B, int H, int W, int cross_class, int max_out,
             float* d_box, float* d_coef_out, int64_t* d_cls, float* d_score, int32_t* d_count,
             float* d_proto, void* stream);

/* yb_infer from uint8 frames: d_img [B,H,W,3] BGR uint8 is FastBaseTransform'ed (as yb_fast_base_transform with
 * img_is_u8 = 1, out_h, out_w, mode, h_mean_bgr, h_std_bgr; NULL = MEANS / STD) and run through the network and Detect
 * as yb_infer(out_h, out_w) does, with the same outputs, bit for bit.  In the tensor-core modes the transform happens
 * inside the stem's operand loader, so no [B,3,out_h,out_w] fp32 input is written; in YB_PREC_F32 it runs as one
 * more kernel in the graph.  The frames are read in place on `stream` (not copied), as the list of B frames
 * yb_infer_frame_list takes, H * W * 3 bytes apart; each (B, out_h, out_w) replays one CUDA graph per transform and
 * NMS mode for any frame size.  YB_ERR_INVALID if d_img is not device memory of the handle's device. */
YB_API int yb_infer_frames(yb_handle* h, const uint8_t* d_img, int B, int H, int W, int out_h, int out_w, int mode,
                           const float* h_mean_bgr, const float* h_std_bgr, int cross_class, int max_out,
                           float* d_box, float* d_coef_out, int64_t* d_cls, float* d_score, int32_t* d_count,
                           float* d_proto, void* stream);

/* yb_infer_frames for a list of B frames of any sizes: h_frames[b] (a host array of device pointers) is a [h, w, 3] BGR
 * uint8 frame with h = h_hw[2b], w = h_hw[2b + 1].  Outputs are yb_infer(out_h, out_w)'s on the B FastBaseTransform'ed
 * frames, bit for bit.  The frames are read in place (not copied); only the B-entry table of pointers, sizes and
 * resize scales is uploaded, so the host arrays may be reused as soon as the call returns.  Nothing depends on the
 * frame sizes: each (B, out_h, out_w) replays one CUDA graph per transform and NMS mode for any mix of them.
 * YB_ERR_INVALID for a null frame pointer, h <= 0 or w <= 0, or a frame that is not device memory of the handle's
 * device. */
YB_API int yb_infer_frame_list(yb_handle* h, const uint8_t* const* h_frames, const int32_t* h_hw, int B, int out_h,
                               int out_w, int mode, const float* h_mean_bgr, const float* h_std_bgr, int cross_class,
                               int max_out, float* d_box, float* d_coef_out, int64_t* d_cls, float* d_score,
                               int32_t* d_count, float* d_proto, void* stream);

/* ---- postprocess (mask assembly) -------------------------------------------------------------- */
/* One image.  proto [ph,pw,k] fp32 NHWC, coef [n,k], box [n,4] relative (NOT modified: the
 * sanitised absolute boxes are written to d_boxes_px as int64 [n,4]).  masks: see yb_mask_format.
 * d_proto_masks (nullable): [n,ph,pw] fp32 cropped sigmoid masks at prototype resolution
 * (the FastMaskIoUNet input, output_utils.py:77-82). */
YB_API int yb_postprocess(yb_handle* h, const float* d_proto, int ph, int pw, int k,
                   const float* d_coef, const float* d_box, int n, int out_h, int out_w,
                   int crop_masks, int mask_format, void* d_masks, int64_t* d_boxes_px,
                   float* d_proto_masks, void* stream);

/* Same for a whole batch in ONE launch (throughput extension; the reference API is per image):
 * proto [B,ph,pw,k], coef [B,n,k], box [B,n,4] (n padded rows per image, e.g. yb_infer's max_out),
 * masks [B,n,...], boxes_px [B,n,4]. */
YB_API int yb_postprocess_batch(yb_handle* h, const float* d_proto, int ph, int pw, int k, const float* d_coef,
                                const float* d_box, int n, int batch, int out_h, int out_w, int crop_masks,
                                int mask_format, void* d_masks, int64_t* d_boxes_px, void* stream);

/* One image of a yb_postprocess_list call (all pointers device memory):
 *   proto [ph,pw,k], coef [n,k], box [n,4] relative: as yb_postprocess's (may be NULL when n == 0);
 *   masks: [n, out_h, out_w] in the call's yb_mask_format (16-byte aligned), or NULL for boxes only;
 *   boxes_px int64 [n,4] (nullable); proto_masks [n,ph,pw] fp32 (nullable; the FastMaskIoUNet input). */
typedef struct {
  const float* proto;
  const float* coef;
  const float* box;
  void* masks;
  int64_t* boxes_px;
  float* proto_masks;
  int32_t n;
  int32_t out_h;
  int32_t out_w;
} yb_post_item;

/* yb_postprocess for a list of B images of any output sizes and row counts, in ONE launch per kernel for the whole
 * list (boxes, prototype-resolution masks, masks): every image's outputs are yb_postprocess's on it, bit for bit.
 * h_items is host memory; it is uploaded into a table the handle owns (stream-ordered behind the handle's previous
 * call) and may be reused as soon as the call returns.  n == 0 is allowed.  YB_ERR_INVALID for a null proto, coef or
 * box with n > 0, n < 0, out_h <= 0 or out_w <= 0, masks not 16-byte aligned, or a pointer that is not device memory
 * of the handle's device. */
YB_API int yb_postprocess_list(yb_handle* h, const yb_post_item* h_items, int B, int ph, int pw, int k,
                               int crop_masks, int mask_format, void* stream);

/* eval.py's --output_coco_json masks for a list of B images, in ONE launch, without materialising them: for every row of
 * every image (rows numbered image by image, n rows each), the pycocotools rleToString string of the mask
 * yb_postprocess_list would produce for that row at out_h x out_w with crop_masks (bilinear, > 0.5), zero-area boxes
 * included: its runs are yb_mask_rle's on yb_postprocess's masks, bit for bit.  h_items as for yb_postprocess_list
 * (proto, coef, box, n, out_h, out_w are read; masks, boxes_px and proto_masks are ignored).
 *   d_runs uint32 [runs_cap]: scratch for the rows' run lengths;  d_chars [chars_cap]: the strings (not
 *   NUL-terminated), row r's at d_chars + d_row_off[r], d_row_len[r] characters (int64 / int32 [rows]).  Rows reserve
 *   their space by atomic add, so the strings need not be in row order.
 *   d_need int64 [2]: the runs and characters the rows asked for.  When either exceeds its cap, the rows that did not
 *   fit have d_row_len -1; calling again with caps of at least d_need[0] and d_need[1] then fits every row (a row whose
 *   runs did not fit asks for 7 characters per run, the most rleToString writes for one).
 * The item table is uploaded into a table the handle owns (stream-ordered behind the handle's previous call); h_items
 * may be reused as soon as the call returns.  B == 0 and n == 0 are allowed.  YB_ERR_INVALID, with nothing written, for
 * a null proto, coef or box with n > 0, n < 0, out_h <= 0 or out_w <= 0, a null output, a negative cap, or a pointer
 * that is not device memory of the handle's device. */
YB_API int yb_coco_rle_list(yb_handle* h, const yb_post_item* h_items, int B, int ph, int pw, int k, int crop_masks,
                            uint32_t* d_runs, int64_t runs_cap, char* d_chars, int64_t chars_cap, int64_t* d_row_off,
                            int32_t* d_row_len, int64_t* d_need, void* stream);

/* maskiou_net on [n,1,ph,pw] fp32 masks -> d_maskiou [n] = net(mask)[i, cls[i]];
 * d_cls == NULL: d_maskiou [n, num_classes-1] = net(mask) (FastMaskIoUNet.forward itself).
 * ph and pw must be >= 63, the smallest mask its five unpadded 3x3/2 convs accept (YB_ERR_INVALID otherwise). */
YB_API int yb_maskiou(yb_handle* h, const float* d_proto_masks, int n, int ph, int pw,
               const int64_t* d_cls, float* d_maskiou, void* stream);

/* ---- either side of the path: frame preparation and eval.py's result consumers ---------------------- */
/* FastBaseTransform.forward: d_img [B,H,W,3] BGR (uint8 when img_is_u8, else fp32 0..255, the
 * reference's `.float()` frame) -> bilinear resize to [out_h,out_w] (align_corners=False) -> transform
 * `mode` with h_mean_bgr / h_std_bgr (3 host floats each; NULL = MEANS / STD of data/config.py:28-29)
 * -> RGB -> d_out [B,3,out_h,out_w] fp32, i.e. exactly yb_forward's input. */
YB_API int yb_fast_base_transform(yb_handle* h, const void* d_img, int img_is_u8, int B, int H, int W,
                                  int out_h, int out_w, int mode, const float* h_mean_bgr,
                                  const float* h_std_bgr, float* d_out, void* stream);

/* 0/1 masks [rows, w] (YB_MASK_F32 or YB_MASK_U8; value > 0.5 -> 1) -> YB_MASK_BITS rows of
 * ceil(w/32) words (padding bits zero).  For ground-truth masks that arrive from the host. */
YB_API int yb_pack_mask_bits(yb_handle* h, const void* d_in, int in_format, int64_t rows, int w,
                             uint32_t* d_bits, void* stream);

/* mask_iou on bit-packed masks: a [n, words], b [m, words] (words = h * ceil(w/32), padding bits
 * zero) -> d_iou [n, m] = |a&b| / (|a| + |b| - |a&b|), or |a&b| / |a| when iscrowd (box_utils.py:113;
 * 0/0 = NaN like the reference). */
YB_API int yb_mask_iou(yb_handle* h, const uint32_t* d_a, int n, const uint32_t* d_b, int m, int64_t words,
                       int iscrowd, float* d_iou, void* stream);

/* jaccard: a [n,4], b [m,4] x1y1x2y2 -> d_iou [n,m] (box_utils.py:54-79). */
YB_API int yb_box_iou(yb_handle* h, const float* d_a, int n, const float* d_b, int m, int iscrowd,
                      float* d_iou, void* stream);

/* COCO run-length encoding of n masks [n,h,w] in `mask_format`: runs in column-major order, alternating
 * 0-runs / 1-runs starting with zeros (counts[0] == 0 when the first pixel is set) -- the `cnts` array
 * of pycocotools' rleEncode.  d_counts [n, cap] uint32, d_nruns [n]: number of runs, or -(needed) when
 * cap was too small for that mask (its counts are then undefined). */
YB_API int yb_mask_rle(yb_handle* h, const void* d_masks, int mask_format, int n, int mask_h, int mask_w,
                       uint32_t* d_counts, int64_t cap, int32_t* d_nruns, void* stream);

/* prep_metrics' matching loop for one image (eval.py:431-509), one launch, no host synchronisation.
 * d_box_iou / d_mask_iou [n,g] and d_crowd_box_iou / d_crowd_mask_iou [n,num_crowd] are the fp32 IoU caches (nullable
 * when g or num_crowd is 0); d_cls int64 [n] detection classes; d_box_score / d_mask_score fp32 [n] (the same pointer
 * twice for a plain score); d_gt_cls / d_crowd_cls int32 [g] / [num_crowd]; h_thresholds: T host doubles.
 * Detections are matched in the stable descending order of their score (box, then mask by mask score with ties in box
 * order), a match needs (double)iou > threshold, an unmatched detection whose crowd IoU exceeds the threshold is not
 * recorded.  Writes 2*T*n records, [type (0 box, 1 mask)][threshold][rank], to d_rec_score (fp32 score) and d_rec_tag
 * (int32: 2 * ((type*T + thr)*C + class) + is_true, or -1 for a crowd hit); the caller places each image's records
 * behind the previous image's, which makes every cell's records the reference's push order.  Adds the per-class
 * ground-truth counts to d_counts int64 [C].  n == 0 does nothing (eval.py:405-406).  A class outside [0, C) sets
 * bit 0 (detection) or bit 1 (ground truth) of d_err.  YB_ERR_INVALID beyond n, g, num_crowd <= 1024, 1 <= T <= 32,
 * 1 <= C <= 2048. */
YB_API int yb_eval_match(yb_handle* h, const float* d_box_iou, const float* d_mask_iou, const float* d_crowd_box_iou,
                         const float* d_crowd_mask_iou, const int64_t* d_cls, const float* d_box_score,
                         const float* d_mask_score, int n, const int32_t* d_gt_cls, int g, const int32_t* d_crowd_cls,
                         int num_crowd, const double* h_thresholds, int T, int C, float* d_rec_score,
                         int32_t* d_rec_tag, int64_t* d_counts, int32_t* d_err, void* stream);

/* One image of a yb_eval_iou_list call (all pointers device memory):
 *   proto [ph,pw,k], coef [n,k], box [n,4] relative, n, out_h, out_w: as yb_post_item's;
 *   boxes_px int64 [n,4]: the pixel boxes yb_postprocess writes for these rows;
 *   gt_bits [g_all, out_h, ceil(out_w/32)] uint32: the ground-truth masks in YB_MASK_BITS rows (padding bits zero);
 *   gt_boxes fp32 [g_all,4]: the ground-truth boxes in pixels; the crowds are the last num_crowd of the g_all rows;
 *   box_iou, mask_iou fp32 [n, g] and crowd_box_iou, crowd_mask_iou fp32 [n, num_crowd], g = g_all - num_crowd: the
 *   outputs (each may be NULL when its side is empty). */
typedef struct {
  const float* proto;
  const float* coef;
  const float* box;
  const int64_t* boxes_px;
  const uint32_t* gt_bits;
  const float* gt_boxes;
  float* box_iou;
  float* mask_iou;
  float* crowd_box_iou;
  float* crowd_mask_iou;
  int32_t n;
  int32_t out_h;
  int32_t out_w;
  int32_t g_all;
  int32_t num_crowd;
} yb_eval_iou_item;

/* prep_metrics' four IoU caches (eval.py:431-445) for a list of B images in ONE launch, straight from the detections:
 * per image, box_iou = jaccard(boxes_px, gt_boxes[:g]), mask_iou = mask_iou(masks, gt[:g]), crowd_box_iou and
 * crowd_mask_iou the same against the crowds with iscrowd, where masks are the YB_MASK_BITS masks yb_postprocess would
 * write for the rows at out_h x out_w with crop_masks (bilinear, > 0.5).  The masks are never written: every cache is
 * yb_box_iou / yb_mask_iou's on yb_postprocess's outputs, bit for bit (0 / 0 = NaN).  Reads the items' proto, coef,
 * box, boxes_px, gt_bits and gt_boxes; writes the four caches and nothing else.  The item table is uploaded into a table
 * the handle owns (stream-ordered behind the handle's previous call); h_items may be reused as soon as the call
 * returns.  No host sync.  B == 0, n == 0 and g_all == 0 are allowed.  YB_ERR_INVALID, with nothing written, for
 * B < 0 or B > 65535, n < 0 or n > 1024, out_h or out_w <= 0, more than 2^28 pixels, num_crowd outside [0, g_all],
 * g or num_crowd > 1024, k not a multiple of 4 or > 128, ph or pw <= 0, a null input or output a non-empty side needs,
 * or a pointer that is not device memory of the handle's device. */
YB_API int yb_eval_iou_list(yb_handle* h, const yb_eval_iou_item* h_items, int B, int ph, int pw, int k,
                            int crop_masks, void* stream);

/* One image of a yb_eval_match_list call (all pointers device memory): the arguments of yb_eval_match for that image
 * (caches, classes, scores, ground-truth and crowd classes, n, g, num_crowd) and rec_offset, the index of the image's
 * first record in the call's d_rec_score / d_rec_tag. */
typedef struct {
  const float* box_iou;
  const float* mask_iou;
  const float* crowd_box_iou;
  const float* crowd_mask_iou;
  const int64_t* cls;
  const float* box_score;
  const float* mask_score;
  const int32_t* gt_cls;
  const int32_t* crowd_cls;
  int64_t rec_offset;
  int32_t n;
  int32_t g;
  int32_t num_crowd;
} yb_eval_match_item;

/* yb_eval_match for a list of B images in ONE launch (one CTA per image): image b's 2*T*n records go to
 * d_rec_score / d_rec_tag + rec_offset, exactly as yb_eval_match would write them at that address, and its non-crowd
 * ground-truth counts are added to d_counts int64 [C]; a class outside [0, C) sets d_err as in yb_eval_match.  An image
 * with n == 0 writes nothing and counts nothing (eval.py:405-406).  Reads the items' caches, classes, scores and
 * ground-truth classes; writes only those records, d_counts and d_err.  The item table is uploaded into a table the
 * handle owns (stream-ordered behind the handle's previous call); h_items and h_thresholds may be reused as soon as the
 * call returns.  No host sync.  YB_ERR_INVALID, with nothing written, for B < 0, any image beyond n, g, num_crowd <=
 * 1024, T outside [1, 32], C outside [1, 2048], a negative rec_offset, a null argument an image with n > 0 needs, or a
 * pointer that is not device memory of the handle's device. */
YB_API int yb_eval_match_list(yb_handle* h, const yb_eval_match_item* h_items, int B, const double* h_thresholds, int T,
                              int C, float* d_rec_score, int32_t* d_rec_tag, int64_t* d_counts, int32_t* d_err,
                              void* stream);

/* Device bytes of the workspace yb_eval_ap needs for num_records records, T thresholds and C classes. */
YB_API int yb_eval_ap_workspace(int64_t num_records, int T, int C, int64_t* bytes);

/* APDataObject.get_ap and is_empty (eval.py:530-581) of every cell of num_records yb_eval_match records in push order:
 * d_ap double [2][T][C] (0 when the cell's count is 0), d_nonempty uint8 [2][T][C].  The records of a cell are sorted
 * stably by descending score, precision and recall are doubles, and the 101 bars are summed in order. */
YB_API int yb_eval_ap(yb_handle* h, const float* d_rec_score, const int32_t* d_rec_tag, int64_t num_records,
                      const int64_t* d_counts, int T, int C, void* d_work, int64_t work_bytes, double* d_ap,
                      uint8_t* d_nonempty, void* stream);

/* Multi-GPU detection gather (the analogue of CustomDataParallel.gather, eval.py:630-634): packs yb_infer / yb_detect's
 * padded outputs of B images into one fp32 record per image, d_rec [B, 1 + M*(6+k)] =
 * [count, cls[M], score[M], box[M*4], coef[M*k]], so that a global batch needs ONE all_gather (NCCL, by the caller). */
YB_API int yb_pack_detections(yb_handle* h, const float* d_box, const float* d_coef, const int64_t* d_cls,
                              const float* d_score, const int32_t* d_count, int B, int M, int k, float* d_rec,
                              void* stream);

/* prep_display's mask blend: d_img [h,w,3] fp32 (0..255 when img_is_255, else 0..1), n masks in
 * `mask_format` in drawing order, d_colors [n,3] fp32 0..1, alpha = mask_alpha ->
 * d_out [h,w,3] uint8 = (blend * 255).byte()  (eval.py:186-209,226). */
YB_API int yb_display_blend(yb_handle* h, const float* d_img, int img_is_255, const void* d_masks,
                            int mask_format, int n, int img_h, int img_w, const float* d_colors, float alpha,
                            uint8_t* d_out, void* stream);

/* One frame of a yb_render_list call (all pointers device memory):
 *   frame [h,w,3] BGR, uint8 or fp32 0..255 (the call's frame_is_u8); out [h,w,3] uint8;
 *   proto [ph,pw,k], coef [n,k], box [n,4] relative, cls int64 [n]: as yb_postprocess's; proto NULL draws no masks
 *   (cfg.eval_mask_branch off) but still selects the rows;
 *   score [n]: the ranking scores (maskiou-rescored for YOLACT++), det_score [n]: Detect's scores, which the
 *   score_threshold filter reads (may equal score);
 *   sel_n int32 [1], sel_cls int64 [top_k], sel_score fp32 [top_k], sel_box int64 [top_k,4] (each nullable): the drawn
 *   rows in drawing order (pixel boxes at h x w), zero past sel_n. */
typedef struct {
  const void* frame;
  uint8_t* out;
  const float* proto;
  const float* coef;
  const float* box;
  const int64_t* cls;
  const float* score;
  const float* det_score;
  int32_t* sel_n;
  int64_t* sel_cls;
  float* sel_score;
  int64_t* sel_box;
  int32_t n;
  int32_t h;
  int32_t w;
} yb_render_item;

/* prep_display(undo_transform=False) without text or boxes, for a list of B frames of any sizes, in two launches for
 * the whole list.  Per frame: rows with det_score > score_threshold (all rows when score_threshold <= 0), in stable
 * descending order of score (ties to the lower row), the first top_k, cut at the first score < score_threshold; drawn
 * slot j gets palette colour (class_color ? cls : j) * 5 % P (d_palette [P,3] fp32 0..1, BGR); out =
 * (frame / 255 blended with the drawn masks at mask_alpha) * 255, .byte().  The masks are postprocess's
 * (crop_masks, bilinear, > 0.5) and are never written: out equals yb_postprocess + the selection + yb_display_blend,
 * bit for bit.  n == 0 or proto == NULL gives the frame's round trip (frame / 255 * 255).byte().  The item table is
 * uploaded into a table the handle owns (stream-ordered behind the handle's previous call); h_items may be reused as
 * soon as the call returns.  YB_ERR_INVALID for a null frame or out, h or w <= 0, n < 0, a null coef, box, cls, score
 * or det_score with n > 0, top_k < 1, P < 1, or a pointer that is not device memory of the handle's device. */
YB_API int yb_render_list(yb_handle* h, const yb_render_item* h_items, int B, int frame_is_u8, int ph, int pw, int k,
                          int crop_masks, int top_k, float score_threshold, int class_color, float mask_alpha,
                          const float* d_palette, int P, void* stream);

/* Options of yb_render_list_ex; all zero except draw_masks = 1 is yb_render_list.
 *   d_counts int32 [B] (nullable, device memory): frame b's row count, read on the device; each item's n is then only
 *     the capacity (the padded rows of yb_infer_frames' outputs, which the item's pointers address) and rows at or
 *     past d_counts[b] are never read.  No count is read on the host, so the call needs no host sync;
 *   fps_w, fps_h (>= 0): the --display_fps box of eval.py:211-219 (cv2.getTextSize of the fps string): pixel rows
 *     [0, min(h, fps_h + 8)) and columns [0, min(w, fps_w + 8)) are scaled by 0.6 after the mask blend and before
 *     * 255; 0, 0 draws no box;
 *   draw_masks: 0 is --display_masks=False: the rows are selected and the sel_* outputs written, no mask is blended. */
typedef struct {
  const int32_t* d_counts;
  int32_t fps_w;
  int32_t fps_h;
  int32_t draw_masks;
} yb_render_opts;

/* yb_render_list with options (opts NULL: the defaults above).  YB_ERR_INVALID, with nothing written, for everything
 * yb_render_list refuses, a negative fps_w or fps_h, or d_counts that is not device memory of the handle's device. */
YB_API int yb_render_list_ex(yb_handle* h, const yb_render_item* h_items, int B, int frame_is_u8, int ph, int pw,
                             int k, int crop_masks, int top_k, float score_threshold, int class_color,
                             float mask_alpha, const float* d_palette, int P, const yb_render_opts* opts,
                             void* stream);

/* ---- op-level entry points --------------------------------------------------------------------- */
/* Mirrors dcn_v2_forward's argument list (src/dcn_v2.h:9-23); all tensors NCHW fp32 contiguous.
 * input [B,C,H,W], weight [Co,C,kh,kw], bias [Co], offset [B,2*dg*kh*kw,Ho,Wo], mask [B,dg*kh*kw,Ho,Wo],
 * output [B,Co,Ho,Wo].  The narrow contract of the YOLACT++ layers: a 3x3 kernel, isotropic stride, padding and
 * dilation, deformable_group 1 and C % 16 == 0 (YB_ERR_INVALID otherwise).  It runs yb_dcn_forward_ex, bit for bit. */
YB_API int yb_dcn_forward(yb_handle* h, const float* d_input, const float* d_weight, const float* d_bias,
                   const float* d_offset, const float* d_mask, float* d_output,
                   int B, int C, int H, int W, int Co,
                   int kernel_h, int kernel_w, int stride_h, int stride_w, int pad_h, int pad_w,
                   int dilation_h, int dilation_w, int deformable_group, void* stream);

/* Geometry of yb_dcn_forward_ex.  Output size Ho = (H + 2 pad_h - (dilation_h (kernel_h - 1) + 1)) / stride_h + 1,
 * likewise Wo. */
typedef struct {
  int32_t kernel_h, kernel_w;        /* >= 1, kernel_h * kernel_w <= 1024 */
  int32_t stride_h, stride_w;        /* >= 1 */
  int32_t pad_h, pad_w;              /* >= 0 */
  int32_t dilation_h, dilation_w;    /* >= 1 */
  int32_t deformable_group;          /* dg >= 1, C % dg == 0 */
} yb_dcn_params;

/* The whole of dcn_v2_forward's domain (dcn_v2_im2col_cuda.cu:125-195).  Offset channel g*2*kh*kw + 2*tap holds the
 * row offset and + 1 the column offset of tap = i*kw + j in deformable group g; mask channel g*kh*kw + tap; input
 * channel c belongs to group c / (C / dg).  Where it runs, by the handle's precision:
 *   f32    the CUDA-core kernel, any C;
 *   f16tc  the tensor-core kernel when (C / dg) % 64 == 0, else the CUDA-core kernel, which needs (C / dg) % 16 == 0;
 *   f16x3  the tensor-core kernel, which needs (C / dg) % 64 == 0.
 * YB_ERR_INVALID, with the output untouched, for a null pointer (bias may be null), a geometry outside the ranges
 * above, a precision's channel rule, B, C, H, W or Co < 1, or an empty output.  Synchronises `stream`. */
YB_API int yb_dcn_forward_ex(yb_handle* h, const float* d_input, const float* d_weight, const float* d_bias,
                             const float* d_offset, const float* d_mask, float* d_output, int B, int C, int H, int W,
                             int Co, const yb_dcn_params* p, void* stream);

/* Deformable position-sensitive RoI pooling, forward (DeformablePSROIPoolForwardKernel of
 * dcn_v2_psroi_pooling_cuda.cu), fp32, one thread per output element.  input NCHW [N,C,H,W], rois [R,5] (batch index,
 * x1, y1, x2, y2 in input-image pixels), trans [R, 2*num_classes, part_size, part_size] (ignored, and may be null,
 * when no_trans; num_classes is then 1), output [R, output_dim, pooled, pooled], count (nullable) the same shape: the
 * samples each bin averaged.  Output channel ctop of bin (ph, pw) reads input channel
 * (ctop * group_size + gh) * group_size + gw.  YB_ERR_INVALID, with nothing written, for a null input, rois, output or
 * (unless no_trans) trans, N, H, W < 1 or R < 0, C != output_dim * group_size^2, num_classes < 1 or
 * output_dim % num_classes != 0, a non-positive pooled, group_size, part_size or sample_per_part, or a RoI whose batch
 * index is not finite or, truncated to an integer as the reference does, outside [0, N).  Synchronises `stream` (the
 * batch indices are checked on the host). */
YB_API int yb_dcn_psroi_pool(yb_handle* h, const float* d_input, const float* d_rois, const float* d_trans,
                             float* d_output, float* d_count, int N, int C, int H, int W, int R, int no_trans,
                             int num_classes, float spatial_scale, int output_dim, int group_size, int pooled,
                             int part_size, int sample_per_part, float trans_std, void* stream);

/* Single convolution through the same kernels the network uses (test / microbench hook).
 * x NCHW fp32 [B,Ci,H,W], w OIHW fp32 (host), bias fp32[Co] (host, nullable),
 * residual NCHW fp32 [B,Co,Ho,Wo] (device, nullable), y NCHW fp32 [B,Co,Ho,Wo].
 * act: 0 none, 1 relu, 2 tanh, 3 leaky_relu(0.1).  precision: 0 fp32 CUDA cores, 1 fp16 tensor cores (YB_PREC_F16TC),
 * 2 fp16 CUDA cores, 3 split-precision tensor cores (YB_PREC_F16X3).
 * iters > 1 repeats the conv kernel and returns the mean kernel time (ms) in *ms (nullable). */
YB_API int yb_conv2d(yb_handle* h, const float* d_x, const float* h_w, const float* h_bias,
              const float* d_residual, float* d_y, int B, int Ci, int H, int W, int Co,
              int kh, int kw, int stride, int pad, int act, int precision, int iters,
              float* ms, void* stream);

/* The cases of the network's convolutions yb_conv2d cannot express (a zeroed struct = none of them). */
typedef struct {
  int32_t res_after_act;         /* y = act(conv) + residual (Darknet blocks) instead of act(conv + residual) */
  int32_t y_f32;                 /* precision 1, 2 or 3: fp32 output straight from the epilogue */
  int32_t cin_pad;               /* x has max(Ci, cin_pad) channels; the weights get zero rows for the extra ones */
  int32_t cout_pad;              /* precision 1 or 3: the output has max(Co, cout_pad) channels, zeros beyond Co */
  int32_t y_pix_stride;          /* fp32 output: elements from one output pixel to the next (>= Co; 0 = Co) */
  int32_t poison;                /* fill d_y with 0xff bytes (fp16 and fp32 NaN) before the launch */
  int32_t nseg;                  /* precision 1 or 3, 0..3: fused prediction head.  Output channels */
  int32_t seg_begin[3];          /*   [seg_begin[i], seg_end[i]) (ascending, disjoint, within Co) go to the fp32 */
  int32_t seg_end[3];            /*   device tensor seg_y[i] at b * seg_batch_stride[i] + pixel * seg_pix_stride[i] */
  int32_t seg_act[3];            /*   + channel - seg_begin[i], with activation seg_act[i]; other channels are not */
  int32_t seg_pix_stride[3];     /*   stored; act and d_y are ignored */
  int64_t seg_batch_stride[3];
  float* seg_y[3];
} yb_conv_opts;

/* yb_conv2d with options, and the output in the kernel's own layout: d_y is NHWC [B,Ho,Wo,Cp] (Cp = max(Co, cout_pad);
 * device, 16-byte aligned) of fp32 (precision 0, or y_f32; [B,Ho,Wo,y_pix_stride] when that is set), fp16 (precision
 * 1 and 2) or, in precision 3, hi / lo fp16 pairs [B,Ho,Wo,hi(Cp) | lo(Cp)] whose value is hi + lo * 2^-11.  The residual is
 * NCHW fp32 [B,Co,Ho,Wo] as in yb_conv2d.  Precision 1 and 3 with Ci == 3 and the network's stem shapes
 * (7x7/2 pad 3 -> 64, 3x3/1 pad 1 -> 32) run the tensor-core stem kernel, cout_pad its zero-padded channels.  The
 * YB_CONV2D_* tiling switches apply as in yb_conv2d.  opts is nullable. */
YB_API int yb_conv2d_ex(yb_handle* h, const float* d_x, const float* h_w, const float* h_bias,
                        const float* d_residual, void* d_y, int B, int Ci, int H, int W, int Co, int kh, int kw,
                        int stride, int pad, int act, int precision, const yb_conv_opts* opts, void* stream);

/* One launch of the network's max pool or bilinear resample (test hook), in the kernels' own layout: d_x [B,H,W,C],
 * d_add (nullable) and d_y [B,Ho,Wo,C] are NHWC device buffers, 16-byte aligned, of fp32 (precision 0), fp16
 * (precision 1) or hi / lo fp16 pairs [.., hi(C) | lo(C)] whose value is hi + lo * 2^-11 (precision 3).
 *   YB_RESAMPLE_MAXPOOL:  3x3 / stride 2 / pad 1 with -inf padding (nn.MaxPool2d); Ho = (H - 1) / 2 + 1 (likewise Wo),
 *                         no add, no relu.
 *   YB_RESAMPLE_BILINEAR: F.interpolate(size=(Ho, Wo), mode='bilinear', align_corners=False), + add, then ReLU when
 *                         relu; the scale is in / out, as the network's FPN and protonet resamples use it.
 * YB_ERR_INVALID, with nothing launched, for another op or precision, C not a multiple of 4 (fp32) or 8 (fp16), or a
 * max pool with another output size, an add or relu.  Asynchronous on `stream`. */
#define YB_RESAMPLE_MAXPOOL 0
#define YB_RESAMPLE_BILINEAR 1
YB_API int yb_resample_ex(yb_handle* h, int op, int precision, const void* d_x, const void* d_add, void* d_y, int B,
                          int H, int W, int C, int Ho, int Wo, int relu, void* stream);

/* ---- introspection ----------------------------------------------------------------------------- */
/* Kernel launches issued by this handle since creation (bench.py's gpu_launches). */
YB_API int64_t yb_launch_count(yb_handle* h);
/* Device time (ms) of the conv stack vs the rest of the last yb_forward, measured with CUDA
 * events on `stream` when profiling was enabled with yb_set_profiling(h,1). */
YB_API int yb_set_profiling(yb_handle* h, int enable);
YB_API int yb_last_forward_ms(yb_handle* h, float* total_ms, float* conv_ms);
/* Per-op CSV ("layer name,ms\n") of the last profiled yb_forward (yb_set_profiling(h,1)). */
YB_API int yb_last_forward_profile(yb_handle* h, char* buf, int64_t cap);
/* Enable/disable CUDA-graph replay of yb_forward (default on). */
YB_API int yb_set_graphs(yb_handle* h, int enable);
/* Host-only mirror of the chain kernel's dependency arithmetic (csrc/tc_conv.cu; no device needed): for a k x k / stride /
 * pad convolution over a B x Hin x Win tensor written by a flattened (1x1 stride 1) or 2-D tiled producer layer, the
 * tilings of both layers and the inclusive range of producer M tiles that consumer M tile `m` waits for.
 * out[14] = consumer {flat, tw, th, tiles_x, tiles_y, m_tiles}, producer {same six}, first, last. */
YB_API int yb_debug_chain_deps(int B, int Hin, int Win, int k, int stride, int pad, int producer_flat, int m, int32_t* out);

/* ---- plan files ---------------------------------------------------------------------------------
 * A handle plans every network input shape it meets by timing: the tensor-core tiling of each layer shape, and for
 * each run of consecutive convolutions whether one chain launch beats the separate launches.  A plan file records
 * these decisions as text; a handle that loads one takes them from the file and times nothing the file covers, so it
 * runs the same kernels, and computes the same bits, as the handle that wrote it (same file, build and GPU model).
 * The header names the build (yb_build_id), the device name, compute capability and SM count, the precision and the
 * switches that change the candidate set (stream-K candidates, YB_CHAIN, programmatic dependent launch).
 *
 * yb_save_plans writes every decision the handle holds (timed or loaded), sorted, so saving right after a load writes
 * the loaded file's bytes.  yb_load_plans merges a file into the handle's table, all or nothing: YB_ERR_INVALID, with
 * the handle untouched and yb_last_error() naming the field, for an unreadable, truncated or malformed file, another
 * format version or build, a header field that differs from this handle's, or an entry that disagrees with a decision
 * the handle already made.  Shapes the file lacks are timed as usual and added to the table.  yb_create loads the
 * file named by the environment variable YB_PLANS when it exists (a refused file is reported on stderr and ignored).
 * yb_plan_stats: decisions made by timing, and plan decisions taken from a loaded file (every use counts), since
 * the handle was created. */
YB_API int yb_save_plans(yb_handle* h, const char* path);
YB_API int yb_load_plans(yb_handle* h, const char* path);
YB_API int yb_plan_stats(yb_handle* h, int64_t* timed, int64_t* loaded);
/* Build id of the compiled kernels: a hash of the CUDA sources and compiler flags, the plan file's `build` field. */
YB_API const char* yb_build_id(void);
/* Host-only (no device needed): parses the plan file at `path` and checks its format, version and build id -- the
 * checks yb_load_plans makes before it compares the header with a handle.  When out_path is not NULL, writes the
 * parsed file back there as yb_save_plans would.  YB_ERR_INVALID, naming the line and field, otherwise. */
YB_API int yb_check_plans(const char* path, const char* out_path);

#ifdef __cplusplus
}
#endif
#endif /* YOLACT_B200_H_ */
