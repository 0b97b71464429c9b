// Launcher declarations for every kernel of the path.  One launcher == one kernel launch
// (each bumps LaunchCounter).  All launchers are asynchronous on `stream`.
#pragma once
#include <vector>
#include "common.cuh"

namespace yb {

// -------------------------------------------------------------------------------------------
// Convolution problem description shared by the SIMT and the tensor-core (wgmma) kernels.
// Activations are NHWC.  Output addressing is  y[b * y_batch_stride + pix * y_pix_stride + c]
// (elements), which lets the 5 head levels write straight into the concatenated
// [B, P, D] tensors the reference builds with permute+view+cat (yolact.py:169-173,633-634).
// -------------------------------------------------------------------------------------------
struct ConvProblem {
  int B = 0, H = 0, W = 0, Cin = 0;
  int Ho = 0, Wo = 0, Cout = 0;
  int KH = 1, KW = 1, stride = 1, pad = 0;
  int act = ACT_NONE;
  const void* x = nullptr;         // NHWC (T) or, when x_nchw_f32, NCHW fp32 (network input)
  int x_nchw_f32 = 0;
  void* y = nullptr;
  int y_f32 = 0;                   // output element type is float even when activations are half
  int64_t y_batch_stride = 0;      // elements
  int y_pix_stride = 0;            // elements
  const float* bias = nullptr;     // [Cout] fp32 (BN folded), nullable
  const void* residual = nullptr;  // dense NHWC [B,Ho,Wo,Cout], activation dtype, nullable
  int res_after_act = 0;           // 1: y = act(conv) + residual (DarkNetBlock, backbone.py:246-247)
  // split precision (tensor-core kernel only, YB_PREC_F16X3): x / residual / half outputs are [hi(C) | lo(C)] fp16 pairs
  // per pixel (y_pix_stride and y_batch_stride count halfs and include both planes), weights are packed
  // [tap][Cout][hi(Cin) | lo(Cin)] and pre-multiplied by 1 / out_scale (a power of two)
  int split = 0;
  float out_scale = 1.f;
  // fused prediction head (tensor-core kernel only): output channels [seg_begin, seg_end) of segment i go to the
  // fp32 tensor seg_y[i] with its own strides and activation; y / y_* are ignored when nseg > 0
  int nseg = 0;
  int seg_begin[3] = {0, 0, 0}, seg_end[3] = {0, 0, 0}, seg_ps[3] = {0, 0, 0}, seg_act[3] = {0, 0, 0};
  int64_t seg_bs[3] = {0, 0, 0};
  float* seg_y[3] = {nullptr, nullptr, nullptr};
};

// Output size of a k-tap window with stride s and padding p over h inputs, as nn.Conv2d / nn.MaxPool2d compute it.  0
// when the padded input is shorter than the window, which nn.Conv2d refuses: C's truncating division alone would give
// 1 there (a 2-pixel input to a 3x3/2 conv), and the kernel would read the missing rows as zeros.
inline int conv_out(int h, int k, int s, int p) { return h + 2 * p < k ? 0 : (h + 2 * p - k) / s + 1; }

enum SimtTypes : int {
  SIMT_F32 = 0,        // x float (NHWC or NCHW), w float, y float
  SIMT_F16,            // x half, w half, y half (or float when y_f32)
};

// w: [KH*KW*Cin][Cout], element type float (SIMT_F32*) or half (SIMT_F16)
void launch_simt_conv(const ConvProblem& p, const void* w, int types, cudaStream_t stream,
                      LaunchCounter* lc);

// ---- wgmma implicit-GEMM convolution (fp16 in, fp32 accumulate) ------------------------------
struct TcConvPlan;  // opaque: tensor maps + tiling; built once per (layer, shape, pointers)
int device_sms();   // SMs of the current device
// The tiling of a tensor-core conv plan.  As a request to tc_conv_plan_create every field is an override, 0 = heuristic;
// tc_conv_plan_tiling returns what a plan resolved to, which replayed as a request gives the same plan.
struct TcTiling {
  int bn = 0;             // N tile in {32, 64, 128, 256}
  int stages = 0;         // caps the pipeline depth
  int grid = 0;           // caps the number of (persistent) CTAs, counted as CTAs (a pair plan's grid is even);
                          // default device_sms() = one per SM
  int pair = 0;           // > 0: CTA pairs (cluster of 2; each CTA loads half the weight tile and multicasts it to both)
  int mma_groups = 0;     // 2: two MMA warpgroups (384 threads)
  int pdl_friendly = 0;   // > 0: plan sized for 2 CTAs/SM + programmatic dependent launch
  int stream_k = 0;       // > 0: stream-K (needs tc_conv_plan_set_sk_workspace before launch)
  int chain = 0;          // > 0: a chain-kernel plan (residual read from global memory in every mode)
};
// "BN=128 st=4 g=132 pair epi2 pdlf sk": names a tiling in op names, and keys the autotuner's dedupe set
std::string tc_tiling_str(const TcTiling& t);
// w_packed: device half [KH*KW][Cout][Cin] ([KH*KW][Cout][2*Cin] when p.split). Requires Cin % 64 == 0.
TcConvPlan* tc_conv_plan_create(const ConvProblem& p, const __half* w_packed, const TcTiling& want = {});
TcTiling tc_conv_plan_tiling(const TcConvPlan* plan);
size_t tc_conv_sk_workspace_bytes();
void tc_conv_plan_set_sk_workspace(TcConvPlan* plan, void* ws);
void tc_conv_plan_set_pdl(TcConvPlan* plan, int enable);   // programmatic dependent launch (prologue overlap)
void tc_conv_plan_destroy(TcConvPlan* plan);
bool tc_conv_supported(const ConvProblem& p);
void launch_tc_conv(const TcConvPlan* plan, cudaStream_t stream, LaunchCounter* lc);
// A run of consecutive layers (each reading the previous one's output) in ONE persistent launch with per-tile
// dependency counters instead of kernel boundaries (tc_conv.cu, "chain kernel"); the plans must outlive the chain
struct TcChain;
bool tc_conv_plan_chainable(const TcConvPlan* plan);
TcChain* tc_chain_create(const std::vector<const TcConvPlan*>& plans, const std::vector<int>& dep_a, const std::vector<int>& dep_r);
void tc_chain_destroy(TcChain* chain);
int tc_chain_layers(const TcChain* chain);
bool tc_chain_graph_ok(const TcChain* chain);
void tc_chain_print_stats(TcChain* chain, const char* name);
void tc_chain_debug_deps(int B, int Hin, int Win, int k, int stride, int pad, int producer_flat, int m, int32_t* out);
void launch_tc_chain(const TcChain* chain, cudaStream_t stream, LaunchCounter* lc);

// ---- stem on the tensor cores (3-channel NCHW fp32 frame -> NHWC fp16) -------------------------------
struct StemTcPlan;
bool stem_tc_supported(int ks, int stride, int pad, int cin, int cout);
int stem_tc_kpad(int ks);   // K = 3*ks*ks rounded up to 64
// w_packed: device half [cout][kpad], k = c*ks*ks + r*ks + s (OIHW flattening), zero padded
// split: w_packed is [cout][hi(kpad) | lo(kpad)] scaled by 1 / out_scale, y is [.., hi(cout) | lo(cout)]; the split 7x7
// stem runs two worker threads per output pixel
StemTcPlan* stem_tc_plan_create(const float* x_nchw, const __half* w_packed, const float* bias, __half* y, int B,
                                int H, int W, int ks, int stride, int pad, int cout, int act, int split = 0,
                                float out_scale = 1.f, int cpad = 0);   // cpad > cout: zero-padded output pixels
// The same stem reading a list of uint8 BGR frames instead: FastBaseTransform to the network's H x W (transform
// `mode`, BGR mean / std) happens in the loader.  Image b's frame, size and scales come from d_table[b] (device,
// net_stem's B entries), read at launch time, so the same plan (and graph) serves any frame sizes the table holds.
// Weights, output and shapes are net_stem's.
StemTcPlan* stem_tc_plan_create_frame_list(const StemTcPlan* net_stem, const FrameRef* d_table, int mode,
                                           const float* mean_bgr, const float* std_bgr);
void stem_tc_plan_destroy(StemTcPlan* plan);
void launch_stem_tc(const StemTcPlan* plan, cudaStream_t stream, LaunchCounter* lc);

// ---- pointwise -------------------------------------------------------------------------------
// `split` (T = __half only): tensors are split-precision [hi(C) | lo(C)] pixel pairs (YB_PREC_F16X3).
// 3x3 stride-2 pad-1 max pool, NHWC (backbone.py:80)
template <typename T>
void launch_maxpool3x3s2(const T* x, T* y, int B, int H, int W, int C, int Ho, int Wo,
                         cudaStream_t stream, LaunchCounter* lc, int split = 0);
// y = bilinear(x -> [Ho,Wo], align_corners=False) (+ add), NHWC.  scale_h/scale_w are the
// source/destination ratios PyTorch uses (in/out, or 1/scale_factor).  relu: clamp at 0.
// The ratio F.interpolate(size=out) uses for in -> out; for out = 2 * in it is exactly 1 / scale_factor = 0.5.
inline float bilinear_scale(int in, int out) { return (float)in / (float)out; }
template <typename T>
void launch_upsample_bilinear(const T* x, const T* add, T* y, int B, int H, int W, int C, int Ho,
                              int Wo, float scale_h, float scale_w, int relu, cudaStream_t stream,
                              LaunchCounter* lc, int split = 0);
// layout / dtype conversion between the kernels' NHWC(T) and the API's NCHW fp32
template <typename T>
void launch_nhwc_to_nchw_f32(const T* x, float* y, int B, int H, int W, int C, cudaStream_t stream,
                             LaunchCounter* lc, int split = 0);
template <typename T>
void launch_nchw_f32_to_nhwc(const float* x, T* y, int B, int C, int H, int W, cudaStream_t stream,
                             LaunchCounter* lc, int split = 0);
void launch_softmax_rows(const float* in, float* out, int64_t rows, int cols, cudaStream_t stream,
                         LaunchCounter* lc);
void launch_fill_u32(uint32_t* p, uint32_t v, int64_t n, cudaStream_t stream, LaunchCounter* lc);

// ---- Detect ------------------------------------------------------------------------------------
struct DetectWorkspace {
  // all device pointers, sized by detect_workspace_bytes
  float* scoresT = nullptr;     // [B][C-1][P]  compacted, class-major
  int32_t* cand_prior = nullptr;  // [B][P]
  int32_t* cand_cls = nullptr;    // [B][P]  argmax fg class per prior (cross-class mode)
  int32_t* cand_count = nullptr;  // [B]
  float* pool_score = nullptr;    // [B][C-1][top_k]
  int32_t* pool_prior = nullptr;  // [B][C-1][top_k]
  float* pool_box = nullptr;      // [B][C-1][top_k][4]
  int32_t* pool_n = nullptr;      // [B][C-1]  kept per class (entries are flagged, see kernel)
};
size_t detect_workspace_bytes(int B, int64_t P, int num_classes, int top_k);
void detect_workspace_bind(DetectWorkspace* ws, void* base, int B, int64_t P, int num_classes,
                           int top_k);
struct DetectParams {
  int B = 0;
  int64_t P = 0;
  int num_classes = 81;
  int mask_dim = 32;
  int top_k = 200;
  float conf_thresh = 0.05f;
  float nms_thresh = 0.5f;
  int max_dets = 100;
  int conf_is_logits = 0;
  int cross_class = 0;          // yb_nms_mode
  int second_threshold = 0;     // fast_nms(second_threshold=True), detection.py:160-161
  float max_size = 550.f;       // cfg.max_size: box scale of traditional_nms (detection.py:194)
  int max_out = 100;
};
void launch_detect(const DetectParams& dp, const float* loc, const float* conf, const float* coef,
                   const float* priors, const DetectWorkspace& ws, float* box, float* coef_out,
                   int64_t* cls, float* score, int32_t* count, cudaStream_t stream,
                   LaunchCounter* lc);

// ---- mask assembly -----------------------------------------------------------------------------
// The images of one postprocess call: a table of B items in device memory (yb_postprocess_list), or, with table ==
// nullptr, a dense batch whose image z is base with every pointer advanced by z times its step (elements, or bytes
// for masks).  Passed by value to the kernels.
struct PostSrc {
  const yb_post_item* table;
  yb_post_item base;
  long long proto_step, coef_step, box_step, masks_step_bytes, boxes_px_step, pm_step;
};
// the dense source of a batch of images like `first`: proto [B,ph,pw,k], coef [B,n,k], box [B,n,4], masks [B,n,...],
// boxes_px [B,n,4], proto_masks [B,n,ph,pw]
PostSrc dense_post_src(const yb_post_item& first, int ph, int pw, int k, int mask_format);
// One launch per kernel for the B images of src: boxes (when an item has boxes_px), prototype-resolution masks (when
// an item has proto_masks), masks (when an item has masks).  h_items is the host view the grid is sized from: the
// table's B entries, or the one dense item.
void launch_mask_assembly(const PostSrc& src, const yb_post_item* h_items, int B, int ph, int pw, int k, int crop,
                          int mask_format, cudaStream_t stream, LaunchCounter* lc);
// global max over HxW per (n, c) then gather channel cls[n] (yolact.py:373, output_utils.py:83)
void launch_maxpool_gather(const float* x_nhwc, int n, int H, int W, int C, const int64_t* cls,
                           float* out, cudaStream_t stream, LaunchCounter* lc);

// ---- frame preparation / eval.py consumers (evalops.cu) -----------------------------------------
void launch_fast_base_transform(const void* img, int img_is_u8, int B, int H, int W, int out_h, int out_w, int mode,
                                const float* mean_bgr, const float* std_bgr, float* out, cudaStream_t stream,
                                LaunchCounter* lc);
// the same from a frame list: image b is d_table[b] (device, B entries), uint8, resized to out_h x out_w
void launch_fast_base_transform_list(const FrameRef* d_table, int B, int out_h, int out_w, int mode,
                                     const float* mean_bgr, const float* std_bgr, float* out, cudaStream_t stream,
                                     LaunchCounter* lc);
void launch_pack_mask_bits(const void* in, int in_format, int64_t rows, int w, uint32_t* out, cudaStream_t stream,
                           LaunchCounter* lc);
void launch_mask_iou_bits(const uint32_t* a, int n, const uint32_t* b, int m, int64_t words, int iscrowd, float* out,
                          cudaStream_t stream, LaunchCounter* lc);
void launch_box_iou(const float* a, int n, const float* b, int m, int iscrowd, float* out, cudaStream_t stream,
                    LaunchCounter* lc);
void launch_mask_rle(const void* masks, int mask_format, int n, int h, int w, uint32_t* counts, int64_t cap,
                     int32_t* nruns, cudaStream_t stream, LaunchCounter* lc);
void launch_pack_detections(const float* box, const float* coef, const int64_t* cls, const float* score,
                            const int32_t* count, int B, int M, int k, float* rec, cudaStream_t stream, LaunchCounter* lc);
void launch_display_blend(const float* img, int img_is_255, const void* masks, int mask_format, int n, int h, int w,
                          const float* colors, float alpha, uint8_t* out, cudaStream_t stream, LaunchCounter* lc);

// ---- eval.py's mAP: detection-to-ground-truth matching and get_ap (evalmap.cu) --------------------------------------
constexpr int EVAL_MAX_DETS = 1024, EVAL_MAX_GT = 1024, EVAL_MAX_THRESHOLDS = 32, EVAL_MAX_CLASSES = 2048;
// The images of one eval_match launch, one CTA each: a table of B items in device memory (yb_eval_match_list), or, with
// table == nullptr, the one image `one` (yb_eval_match: passed by value, nothing uploaded).  An item's IoU caches are
// [n,g] / [n,num_crowd] fp32 (nullable when that side is empty); its records go to rec_score / rec_tag + rec_offset.
struct EvalMatchSrc {
  const yb_eval_match_item* table;
  yb_eval_match_item one;
  int T, C;
  double thr[EVAL_MAX_THRESHOLDS];
  float* rec_score;                     // [2][T][n] per image at its rec_offset
  int32_t* rec_tag;                     // [2][T][n]: 2 * cell + is_true, or -1 (crowd hit / bad class)
  int64_t* counts;                      // [C] non-crowd ground truths per class, accumulated
  int32_t* err;                         // bit 0: detection class out of range, bit 1: ground-truth class out of range
};
void eval_check_limits(int n, int g, int num_crowd, int T, int C);
// One launch for the B images of src (h_items: their host view, B entries, or &src.one with B == 1); none when no image
// has detections.
void launch_eval_match(const EvalMatchSrc& src, const yb_eval_match_item* h_items, int B, cudaStream_t stream,
                       LaunchCounter* lc);
// The four IoU caches of the B images of d_items (device; h_items is its host view) straight from the detections, in one
// launch (evaliou.cu); none when no image has both detections and ground truth.
void launch_eval_iou(const yb_eval_iou_item* d_items, const yb_eval_iou_item* h_items, int B, int ph, int pw, int k,
                     int crop, cudaStream_t stream, LaunchCounter* lc);
size_t eval_ap_workspace_bytes(int64_t R, int T, int C);
// R records -> ap [2][T][C] double, nonempty [2][T][C] uint8 (APDataObject.get_ap / is_empty of every cell)
void launch_eval_ap(const float* rec_score, const int32_t* rec_tag, int64_t R, const int64_t* counts, int T, int C,
                    void* work, size_t work_bytes, double* ap, uint8_t* nonempty, cudaStream_t stream, LaunchCounter* lc);

// ---- prep_display's mask overlay from the detections (render.cu) ---------------------------------------------------
// Device bytes of the work table launch_render needs for B images and top_k slots.
size_t render_work_bytes(int B, int top_k);
// Two launches for the B images of d_items (device; h_items is its host view): the selection, then the render of
// every image's drawn masks over its frame.  opts: device row counts (items' n is then the capacity), the fps box and
// draw_masks, as yb_render_list_ex documents them.  work: render_work_bytes(B, top_k) bytes of device memory.
void launch_render(const yb_render_item* d_items, const yb_render_item* h_items, int B, int frame_is_u8, int ph, int pw,
                   int k, int crop, int top_k, float score_threshold, int class_color, float alpha,
                   const float* palette, int P, const yb_render_opts& opts, void* work, cudaStream_t stream,
                   LaunchCounter* lc);

// ---- eval.py's COCO results masks from the detections (cocorle.cu) --------------------------------------------------
// One launch for the B images of d_items (device; h_items is its host view): every row's rleToString string of the mask
// launch_mask_assembly would produce, in the chars arena at row_off[row] (row_len[row] characters, or -1 when an arena
// was too small); need[0] / need[1] = the runs / characters all rows asked for.  Zeroes need first.
void launch_coco_rle(const yb_post_item* d_items, const yb_post_item* h_items, int B, int ph, int pw, int k, int crop,
                     uint32_t* runs, int64_t runs_cap, char* chars, int64_t chars_cap, int64_t* row_off,
                     int32_t* row_len, int64_t* need, cudaStream_t stream, LaunchCounter* lc);

// ---- DCNv2 -------------------------------------------------------------------------------------
// Geometry g (yb_dcn_params: kh x kw taps, tap = i*kw + j, per-axis stride / pad / dilation, dg deformable groups).
// x NHWC (T) [B,H,W,C]; om NHWC fp32 [B,Ho,Wo,3*dg*taps]: the offsets (channel gr*2*taps + 2*tap = dh, + 1 = dw of
// group gr), then the masks (2*dg*taps + gr*taps + tap; logits when mask_logits, dcn_v2.py:118-124) -- for the
// network's 3x3 layers the 27 channels of conv_offset_mask; w: [taps*C][Cout] (T), row tap*C + c; y NHWC (T).
// Fused deformable gather + contraction + bias + activation, any C with C % dg == 0.
template <typename T>
void launch_dcn_simt(const T* x, const float* om, const T* w, const float* bias, T* y, int B, int H,
                     int W, int C, int Ho, int Wo, int Cout, const yb_dcn_params& g, int act,
                     int mask_logits, cudaStream_t stream, LaunchCounter* lc);

// ---- fused DCNv2 on the tensor cores (dcn_tc.cu): gather -> smem A stage -> MMA -> bias/act, no column buffer ----------------
struct DcnTcPlan;
// (C / dg) % 64 == 0: every 64-channel k-block lies inside one deformable group
bool dcn_tc_supported(int C, int Cout, int dg = 1);
// x NHWC half [B,H,W,C] (split: [.., hi(C) | lo(C)]), om as launch_dcn_simt's, w_packed [Cout][taps*C] half with
// k = tap*C + c (split: [Cout][hi(taps*C) | lo(taps*C)] scaled by 1 / out_scale), y NHWC half [B,Ho,Wo,Cout] (split: pairs).
DcnTcPlan* dcn_tc_plan_create(const __half* x, const float* om, const __half* w_packed, const float* bias, __half* y, int B,
                              int H, int W, int C, int Ho, int Wo, int Cout, const yb_dcn_params& g, int act,
                              int mask_logits, int split = 0, float out_scale = 1.f, int bn_override = 0);
void dcn_tc_plan_destroy(DcnTcPlan* plan);
void launch_dcn_tc(const DcnTcPlan* plan, cudaStream_t stream, LaunchCounter* lc);
// The 3x3 geometry of the network's DCN layers (stride s, padding 1, dilation 1, one deformable group).
inline yb_dcn_params dcn_3x3(int stride) { return yb_dcn_params{3, 3, stride, stride, 1, 1, 1, 1, 1}; }

// ---- deformable PS-RoI pooling (dcn_pool.cu), fp32 NCHW, one thread per output element ------------------------------
struct PsroiPoolArgs {
  const float* x;        // [N, C, H, W]
  const float* rois;     // [R, 5]
  const float* trans;    // [R, 2 * num_classes, part, part], unread when no_trans
  float* y;              // [R, output_dim, pooled, pooled]
  float* count;          // same shape, nullable
  int N, C, H, W, R;
  int no_trans, num_classes, output_dim, group_size, pooled, part_size, sample_per_part;
  float spatial_scale, trans_std;
};
void launch_dcn_psroi_pool(const PsroiPoolArgs& a, cudaStream_t stream, LaunchCounter* lc);

}  // namespace yb
