// C ABI (include/yolact_b200.h).  Every entry point converts C++ exceptions into a status code
// and a thread-local message; nothing here computes on the CPU beyond packing weights.
#include <stdlib.h>
#include <string.h>

#include "engine.cuh"

namespace yb {
static thread_local std::string g_last_error;
void set_last_error(const std::string& msg) { g_last_error = msg; }
}  // namespace yb

using namespace yb;

#define YB_API_BEGIN try {
#define YB_API_END                                   \
  }                                                  \
  catch (const yb::Error& e) {                       \
    yb::set_last_error(e.what());                    \
    return e.code;                                   \
  }                                                  \
  catch (const std::exception& e) {                  \
    yb::set_last_error(std::string("internal: ") + e.what()); \
    return YB_ERR_INVALID;                           \
  }                                                  \
  return YB_OK;

namespace {

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) YB_CHECK_CUDA(cudaSetDevice(dev));
  }
  ~DeviceGuard() {
    int cur = -1;
    cudaGetDevice(&cur);
    if (prev >= 0 && cur != prev) cudaSetDevice(prev);
  }
};

// offset [B,2n,HW] + mask [B,n,HW] (NCHW fp32, n = dg * taps) -> om [B,HW,3n]
__global__ void pack_om_kernel(const float* __restrict__ off, const float* __restrict__ msk, float* __restrict__ om,
                               int B, int HW, int n) {
  const int64_t total = (int64_t)B * HW * 3 * n;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int ch = (int)(i % (3 * n));
    int64_t r = i / (3 * n);
    int p = (int)(r % HW);
    int b = (int)(r / HW);
    om[i] = ch < 2 * n ? off[((int64_t)b * 2 * n + ch) * HW + p] : msk[((int64_t)b * n + (ch - 2 * n)) * HW + p];
  }
}

// Every entry point that takes a handle holds its mutex while it enqueues work (the handle's plans, launch counter
// and lazily grown workspaces are not thread-safe by themselves).  Entry points that run on the handle's SHARED device
// buffers (executor activations, Detect workspace, scratch) additionally order themselves on the device behind the
// previous such call when it was issued on a different stream -- eval.py's ThreadPool callers (eval.py:793-827) may
// drive one net from several threads / streams; results are then serialised, never corrupted.
struct CallGuard {
  yb_handle* h;
  DeviceGuard dg;
  std::unique_lock<std::recursive_mutex> lk;
  cudaStream_t stream = nullptr;
  bool chain = false;
  explicit CallGuard(yb_handle* h_) : h(h_), dg(h_->device), lk(h_->mu) {}
  static bool capturing(cudaStream_t s) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(s, &st) != cudaSuccess) {
      cudaGetLastError();
      return true;
    }
    return st != cudaStreamCaptureStatusNone;
  }
  CallGuard(yb_handle* h_, cudaStream_t s) : h(h_), dg(h_->device), lk(h_->mu), stream(s), chain(true) {
    // (a stream the CALLER is capturing neither waits on nor records the handle's event: ordering is the caller's graph)
    if (h->ev_last && h->has_last && h->last_stream != s && !capturing(s)) cudaStreamWaitEvent(s, h->ev_last, 0);
  }
  ~CallGuard() {
    if (!chain || capturing(stream)) return;
    if (!h->ev_last && cudaEventCreateWithFlags(&h->ev_last, cudaEventDisableTiming) != cudaSuccess) {
      cudaGetLastError();
      h->ev_last = nullptr;
      return;
    }
    if (cudaEventRecord(h->ev_last, stream) == cudaSuccess) {
      h->last_stream = stream;
      h->has_last = true;
    } else {
      cudaGetLastError();
    }
  }
};

struct TempPool {  // RAII device temporaries for the op-level hooks
  std::vector<void*> v;
  void* get(size_t bytes) {
    void* p = nullptr;
    YB_CHECK_CUDA(cudaMalloc(&p, std::max<size_t>(bytes, 256)));
    v.push_back(p);
    return p;
  }
  void* put(const PackedWeights& pw) {   // a device copy of packed weights, in whichever element format they hold
    const size_t bytes = pw.f.size() * 4 + pw.h.size() * 2;
    void* p = get(bytes);
    YB_CHECK_CUDA(cudaMemcpy(p, pw.f.empty() ? (const void*)pw.h.data() : pw.f.data(), bytes, cudaMemcpyHostToDevice));
    return p;
  }
  ~TempPool() {
    for (void* p : v) cudaFree(p);
  }
};

// The tensor-core plan of an op-level conv hook, tiled as the YB_CONV2D_* switches ask (unset = the heuristic), with
// its stream-K workspace (zeroed on s) from tp.
TcConvPlan* hook_tc_plan(const ConvProblem& p, const __half* w, TempPool& tp, cudaStream_t s) {
  auto env = [](const char* name) {
    const char* v = getenv(name);
    return v ? atoi(v) : 0;
  };
  TcTiling want;
  want.bn = env("YB_CONV2D_BN");
  want.grid = env("YB_CONV2D_GRID");
  want.pair = env("YB_CONV2D_PAIR");
  want.mma_groups = env("YB_CONV2D_EPI");
  want.pdl_friendly = env("YB_CONV2D_PDL");   // PDL-friendly plan + programmatic dependent launch
  want.stream_k = env("YB_CONV2D_SK");
  TcConvPlan* plan = tc_conv_plan_create(p, w, want);
  if (want.pdl_friendly) tc_conv_plan_set_pdl(plan, 1);
  if (tc_conv_plan_tiling(plan).stream_k) {
    try {
      void* ws = tp.get(tc_conv_sk_workspace_bytes());
      YB_CHECK_CUDA(cudaMemsetAsync(ws, 0, tc_conv_sk_workspace_bytes(), s));
      tc_conv_plan_set_sk_workspace(plan, ws);
    } catch (...) {
      tc_conv_plan_destroy(plan);
      throw;
    }
  }
  return plan;
}

// data/config.py:28-29 (BGR order): the transform's mean / std when the caller passes NULL
const float kMeans[3] = {103.94f, 116.78f, 123.68f};
const float kStd[3] = {57.38f, 57.12f, 58.40f};

inline int grid1d(int64_t n) { return (int)std::min<int64_t>(132 * 16, (n + 255) / 256); }

// The frame inputs are read in place by the network's kernels: YB_ERR_INVALID unless frame is device (or managed)
// memory of the handle's device.
void require_device_frame(const yb_handle* h, const void* frame, const char* msg) {
  cudaPointerAttributes a;
  const bool found = cudaPointerGetAttributes(&a, frame) == cudaSuccess;
  if (!found) cudaGetLastError();   // not a pointer CUDA knows: clear the error, then reject
  YB_REQUIRE(found && (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == h->device, msg);
}

// The list entry points' pointer check: NULL, or device (or managed) memory of the handle's device.
bool on_handle_device(const yb_handle* h, const void* p) {
  if (!p) return true;
  cudaPointerAttributes a;
  const bool found = cudaPointerGetAttributes(&a, p) == cudaSuccess;
  if (!found) cudaGetLastError();   // not a pointer CUDA knows: clear the error, then reject
  return found && (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == h->device;
}

// A yb_post_item table's refusals, named after the entry point `where`, before anything is written or launched.
// with_outputs: the caller writes the items' outputs, so masks must also be 16-byte aligned and masks, boxes_px and
// proto_masks on the handle's device.
void check_post_items(const yb_handle* h, const yb_post_item* h_items, int B, const char* where, bool with_outputs) {
  const std::string w(where);
  auto on_device = [h](const void* p) { return on_handle_device(h, p); };
  for (int b = 0; b < B; ++b) {
    const yb_post_item& it = h_items[b];
    YB_REQUIRE(it.n >= 0 && it.out_h > 0 && it.out_w > 0, w + ": n must be >= 0 and out_h, out_w > 0");
    YB_REQUIRE(it.n == 0 || (it.proto && it.coef && it.box), w + ": null proto, coef or box");
    YB_REQUIRE(!with_outputs || (reinterpret_cast<uintptr_t>(it.masks) & 15) == 0, w + ": masks must be 16-byte aligned");
    YB_REQUIRE(on_device(it.proto) && on_device(it.coef) && on_device(it.box) &&
                   (!with_outputs || (on_device(it.masks) && on_device(it.boxes_px) && on_device(it.proto_masks))),
               w + ": a pointer is not device memory of the handle's device");
  }
}

// Copies a host item table of B entries to the front of buf (at least `bytes` long) on `stream` and returns it.  The
// source is pageable, so the copy is staged before the call returns and the caller may reuse h_items at once.  The
// caller holds a CallGuard on `stream`, so the copy is ordered after the previous call's launches, which have read the
// table before it is overwritten.
template <class T>
T* stage_items(yb::DeviceBuffer& buf, size_t bytes, const T* h_items, int B, void* stream) {
  T* table = static_cast<T*>(buf.get(bytes));
  if (B > 0)
    YB_CHECK_CUDA(cudaMemcpyAsync(table, h_items, (size_t)B * sizeof(T), cudaMemcpyHostToDevice, (cudaStream_t)stream));
  return table;
}

}  // namespace

extern "C" {

int yb_abi_version(void) { return YB_ABI_VERSION; }
const char* yb_last_error(void) { return yb::g_last_error.c_str(); }

int yb_device_count(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) {
    cudaGetLastError();
    yb::set_last_error(std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e));
    return YB_ERR_NO_DEVICE;
  }
  return n;
}

int yb_create(const yb_config* cfg, int device, yb_handle** out) {
  YB_API_BEGIN
  YB_REQUIRE(cfg && out, "yb_create: null argument");
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) {
    cudaGetLastError();
    throw Error(YB_ERR_NO_DEVICE, "yb_create: no CUDA device is visible (this library has no CPU fallback)");
  }
  YB_REQUIRE(device >= 0 && device < n, "yb_create: bad device index");
  cudaDeviceProp prop;
  YB_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
  YB_REQUIRE(prop.major == 9 && prop.minor == 0, "yb_create: this library is built for sm_90a (Hopper H100) only");
  std::unique_ptr<yb_handle> h(new yb_handle());
  h->cfg = *cfg;
  h->device = device;
  h->ops_only = (cfg->backbone == YB_BACKBONE_NONE);
  // defaults: programmatic dependent launch in the single-pass fp16 mode, stream-K candidates in the split mode (whose
  // plans fill the SM, so nothing can become resident early).  Not measured on the H100; YB_SK switches stream-K.
  h->pdl = (cfg->precision == YB_PREC_F16TC);
  h->sk_candidates = (cfg->precision == YB_PREC_F16X3);
  if (const char* sk = getenv("YB_SK")) h->sk_candidates = (atoi(sk) != 0);
  if (const char* ch = getenv("YB_CHAIN")) h->chain_mode = std::min(2, std::max(0, atoi(ch)));
  if (!h->ops_only) {
    YB_REQUIRE(cfg->backbone == YB_BACKBONE_RESNET || cfg->backbone == YB_BACKBONE_DARKNET, "unknown backbone");
    YB_REQUIRE(cfg->num_stages >= 4 && cfg->num_stages <= 5, "num_stages must be 4 or 5");
    YB_REQUIRE(cfg->fpn_features == 256 || cfg->fpn_features % 64 == 0, "fpn_features must be a multiple of 64");
    YB_REQUIRE(cfg->num_scales >= 1 && cfg->num_scales <= 4 && cfg->num_ars >= 1 && cfg->num_ars <= 4, "bad anchors");
    for (int i = 0; i < 3; ++i)
      YB_REQUIRE(cfg->selected_layers[i] >= 0 && cfg->selected_layers[i] < cfg->num_stages, "bad selected_layers");
  }
  YB_REQUIRE(cfg->precision == YB_PREC_F32 || cfg->precision == YB_PREC_F16TC || cfg->precision == YB_PREC_F16X3,
             "unknown precision");
  YB_REQUIRE(cfg->mask_dim % 4 == 0 && cfg->mask_dim > 0, "mask_dim must be a positive multiple of 4");
  DeviceGuard g(device);
  YB_CHECK_CUDA(cudaFree(0));
  // YB_PLANS=<path>: start from a saved plan file when there is one (a network handle whose header it does not match
  // plans by timing, as without it)
  const char* plans = getenv("YB_PLANS");
  if (plans && *plans && !h->ops_only) {
    if (FILE* fp = fopen(plans, "rb")) {
      fclose(fp);
      try {
        h->load_plans(plans);
      } catch (const yb::Error& e) {
        fprintf(stderr, "[yolact_b200] YB_PLANS=%s not loaded: %s\n", plans, e.what());
      }
    }
  }
  *out = h.release();
  YB_API_END
}

int yb_destroy(yb_handle* h) {
  YB_API_BEGIN
  if (h) {
    DeviceGuard dg(h->device);
    cudaDeviceSynchronize();
    delete h;
  }
  YB_API_END
}

int yb_load_weight(yb_handle* h, const char* name, const float* h_data, const int64_t* shape, int ndim) {
  YB_API_BEGIN
  YB_REQUIRE(h && name && h_data && (shape || ndim == 0), "yb_load_weight: null argument");
  YB_REQUIRE(ndim >= 0 && ndim <= 8, "yb_load_weight: bad ndim");
  HostTensor t;
  int64_t n = 1;
  for (int i = 0; i < ndim; ++i) {
    YB_REQUIRE(shape[i] >= 0, "yb_load_weight: negative dim");
    t.shape.push_back(shape[i]);
    n *= shape[i];
  }
  t.data.assign(h_data, h_data + n);
  h->host[name] = std::move(t);
  h->finalized = false;
  YB_API_END
}

int yb_finalize_weights(yb_handle* h) {
  YB_API_BEGIN
  YB_REQUIRE(h, "null handle");
  CallGuard g(h);
  h->finalize();
  YB_API_END
}

int yb_num_priors(yb_handle* h, int img_h, int img_w, int64_t* num_priors, int32_t* level_hw) {
  YB_API_BEGIN
  YB_REQUIRE(h && !h->ops_only, "yb_num_priors: handle has no network");
  int lhw[5][2];
  compute_level_sizes(h->cfg, img_h, img_w, lhw, nullptr, nullptr);
  int64_t P = 0;
  for (int l = 0; l < 5; ++l) {
    P += (int64_t)lhw[l][0] * lhw[l][1] * h->cfg.num_scales * h->cfg.num_ars;
    if (level_hw) {
      level_hw[2 * l] = lhw[l][0];
      level_hw[2 * l + 1] = lhw[l][1];
    }
  }
  if (num_priors) *num_priors = P;
  YB_API_END
}

int yb_priors(yb_handle* h, int img_h, int img_w, float* d_priors, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && !h->ops_only && d_priors, "yb_priors: bad argument");
  CallGuard g(h);
  int lhw[5][2];
  compute_level_sizes(h->cfg, img_h, img_w, lhw, nullptr, nullptr);
  std::vector<float> pri = make_priors_host(h->cfg, lhw);
  YB_CHECK_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  YB_CHECK_CUDA(cudaMemcpy(d_priors, pri.data(), pri.size() * 4, cudaMemcpyHostToDevice));
  YB_API_END
}

int yb_proto_size(yb_handle* h, int img_h, int img_w, int32_t* ph, int32_t* pw) {
  YB_API_BEGIN
  YB_REQUIRE(h && !h->ops_only, "yb_proto_size: handle has no network");
  int lhw[5][2], a, b;
  compute_level_sizes(h->cfg, img_h, img_w, lhw, &a, &b);
  if (ph) *ph = a;
  if (pw) *pw = b;
  YB_API_END
}

int yb_forward(yb_handle* h, const float* d_x, int B, int H, int W, float* d_loc, float* d_conf, float* d_coef,
               float* d_proto, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_x && B > 0 && H > 0 && W > 0, "yb_forward: bad argument");
  YB_REQUIRE(!h->ops_only, "yb_forward: handle has no network");
  CallGuard g(h, (cudaStream_t)stream);   // shared workspaces: ordered behind the previous call
  h->forward(d_x, B, H, W, d_loc, d_conf, d_coef, d_proto, (cudaStream_t)stream);
  YB_API_END
}

int yb_infer(yb_handle* h, const float* d_x, int B, int H, int W, int cross_class, int max_out, float* d_box,
             float* d_coef_out, int64_t* d_cls, float* d_score, int32_t* d_count, float* d_proto, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_x && B > 0 && H > 0 && W > 0, "yb_infer: bad argument");
  YB_REQUIRE(!h->ops_only, "yb_infer: handle has no network");
  YB_REQUIRE(d_box && d_coef_out && d_cls && d_score && d_count, "yb_infer: null output");
  CallGuard g(h, (cudaStream_t)stream);   // shared workspaces: ordered behind the previous call
  h->infer(d_x, B, H, W, cross_class, max_out, d_box, d_coef_out, d_cls, d_score, d_count, d_proto,
           (cudaStream_t)stream);
  YB_API_END
}

int yb_infer_frames(yb_handle* h, const uint8_t* d_img, int B, int H, int W, int out_h, int out_w, int mode,
                    const float* h_mean_bgr, const float* h_std_bgr, int cross_class, int max_out, float* d_box,
                    float* d_coef_out, int64_t* d_cls, float* d_score, int32_t* d_count, float* d_proto,
                    void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_img && B > 0 && H > 0 && W > 0 && out_h > 0 && out_w > 0, "yb_infer_frames: bad argument");
  YB_REQUIRE(!h->ops_only, "yb_infer_frames: handle has no network");
  YB_REQUIRE(d_box && d_coef_out && d_cls && d_score && d_count, "yb_infer_frames: null output");
  YB_REQUIRE(mode >= YB_XFORM_NORMALIZE && mode <= YB_XFORM_NONE, "yb_infer_frames: unknown transform mode");
  require_device_frame(h, d_img, "yb_infer_frames: the frames are not device memory of the handle's device");
  // a frame list whose B entries lie H * W * 3 bytes apart
  std::vector<const uint8_t*> frames(B);
  std::vector<int32_t> hw(2 * (size_t)B);
  for (int b = 0; b < B; ++b) {
    frames[b] = d_img + (size_t)b * H * W * 3;
    hw[2 * b] = H;
    hw[2 * b + 1] = W;
  }
  CallGuard g(h, (cudaStream_t)stream);   // shared workspaces and frame table: ordered behind the previous call
  h->infer_frame_list(frames.data(), hw.data(), B, out_h, out_w, mode, h_mean_bgr ? h_mean_bgr : kMeans,
                      h_std_bgr ? h_std_bgr : kStd, cross_class, max_out, d_box, d_coef_out, d_cls, d_score, d_count,
                      d_proto, (cudaStream_t)stream);
  YB_API_END
}

int yb_infer_frame_list(yb_handle* h, const uint8_t* const* h_frames, const int32_t* h_hw, int B, int out_h, int out_w,
                        int mode, const float* h_mean_bgr, const float* h_std_bgr, int cross_class, int max_out,
                        float* d_box, float* d_coef_out, int64_t* d_cls, float* d_score, int32_t* d_count,
                        float* d_proto, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && h_frames && h_hw && B > 0 && out_h > 0 && out_w > 0, "yb_infer_frame_list: bad argument");
  YB_REQUIRE(!h->ops_only, "yb_infer_frame_list: handle has no network");
  YB_REQUIRE(d_box && d_coef_out && d_cls && d_score && d_count, "yb_infer_frame_list: null output");
  YB_REQUIRE(mode >= YB_XFORM_NORMALIZE && mode <= YB_XFORM_NONE, "yb_infer_frame_list: unknown transform mode");
  for (int b = 0; b < B; ++b) {
    YB_REQUIRE(h_frames[b], "yb_infer_frame_list: null frame pointer");
    YB_REQUIRE(h_hw[2 * b] > 0 && h_hw[2 * b + 1] > 0, "yb_infer_frame_list: frame height and width must be positive");
    require_device_frame(h, h_frames[b], "yb_infer_frame_list: a frame is not device memory of the handle's device");
  }
  CallGuard g(h, (cudaStream_t)stream);   // shared workspaces and frame table: ordered behind the previous call
  h->infer_frame_list(h_frames, h_hw, B, out_h, out_w, mode, h_mean_bgr ? h_mean_bgr : kMeans,
                      h_std_bgr ? h_std_bgr : kStd, cross_class, max_out, d_box, d_coef_out, d_cls, d_score, d_count,
                      d_proto, (cudaStream_t)stream);
  YB_API_END
}

int yb_debug_feature(yb_handle* h, int which, float* d_out, int32_t* chw, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && h->last_exec && which >= 0 && which < 9, "yb_debug_feature: no forward has run / bad index");
  CallGuard g(h, (cudaStream_t)stream);   // shared workspaces: ordered behind the previous call
  const Act& a = h->last_exec->feats[which];
  YB_REQUIRE(a.ptr != nullptr, "yb_debug_feature: feature not available for this backbone");
  if (chw) {
    chw[0] = a.C;
    chw[1] = a.H;
    chw[2] = a.W;
  }
  if (d_out) {
    if (a.f32)
      launch_nhwc_to_nchw_f32<float>((const float*)a.ptr, d_out, a.B, a.H, a.W, a.C, (cudaStream_t)stream, &h->lc);
    else
      launch_nhwc_to_nchw_f32<__half>((const __half*)a.ptr, d_out, a.B, a.H, a.W, a.C, (cudaStream_t)stream, &h->lc,
                                      a.split ? 1 : 0);
  }
  YB_API_END
}

int yb_softmax(yb_handle* h, const float* d_in, float* d_out, int64_t rows, int cols, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_in && d_out && rows >= 0 && cols > 0, "yb_softmax: bad argument");
  CallGuard g(h);
  launch_softmax_rows(d_in, d_out, rows, cols, (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_set_detect_params(yb_handle* h, int top_k, float conf_thresh, float nms_thresh, int max_num_detections) {
  YB_API_BEGIN
  YB_REQUIRE(h, "yb_set_detect_params: null handle");
  YB_REQUIRE(top_k >= 1 && top_k <= 256, "yb_set_detect_params: top_k must be in [1, 256] (one CTA sorts a class)");
  YB_REQUIRE(max_num_detections >= 1 && max_num_detections <= 256, "yb_set_detect_params: max_num_detections must be in [1, 256]");
  YB_REQUIRE(nms_thresh > 0.f, "nms_threshold must be non negative.");   // detection.py:25-26
  CallGuard g(h);
  yb_config& c = h->cfg;
  if (c.nms_top_k == top_k && c.nms_conf_thresh == conf_thresh && c.nms_thresh == nms_thresh &&
      c.max_num_detections == max_num_detections)
    return YB_OK;
  YB_CHECK_CUDA(cudaDeviceSynchronize());
  c.nms_top_k = top_k;
  c.nms_conf_thresh = conf_thresh;
  c.nms_thresh = nms_thresh;
  c.max_num_detections = max_num_detections;
  for (auto& kv : h->execs) kv.second->drop_detect_state();   // workspace sizes and captured graphs depend on them
  YB_API_END
}

int yb_detect(yb_handle* h, const float* d_loc, const float* d_conf, const float* d_coef, const float* d_priors,
              int B, int64_t P, int conf_is_logits, int cross_class, int max_out, float* d_box, float* d_coef_out,
              int64_t* d_cls, float* d_score, int32_t* d_count, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_loc && d_conf && d_coef && d_priors && d_box && d_coef_out && d_cls && d_score && d_count,
             "yb_detect: null argument");
  YB_REQUIRE(B > 0 && P > 0, "yb_detect: empty input");
  CallGuard g(h, (cudaStream_t)stream);   // shared workspaces: ordered behind the previous call
  DetectParams dp;
  dp.B = B;
  dp.P = P;
  dp.num_classes = h->cfg.num_classes;
  dp.mask_dim = h->cfg.mask_dim;
  dp.top_k = h->cfg.nms_top_k;
  dp.conf_thresh = h->cfg.nms_conf_thresh;
  dp.nms_thresh = h->cfg.nms_thresh;
  dp.max_dets = h->cfg.max_num_detections;
  dp.conf_is_logits = conf_is_logits;
  dp.cross_class = cross_class & 0xFF;
  dp.second_threshold = (cross_class & YB_NMS_FLAG_SECOND_THRESHOLD) ? 1 : 0;
  dp.max_size = (float)h->cfg.max_size;
  dp.max_out = max_out;
  YB_REQUIRE(dp.nms_thresh > 0.f, "nms_threshold must be non negative.");  // detection.py:25-26
  void* ws = h->detect_ws.get(detect_workspace_bytes(B, P, dp.num_classes, dp.top_k));
  DetectWorkspace dws;
  detect_workspace_bind(&dws, ws, B, P, dp.num_classes, dp.top_k);
  launch_detect(dp, d_loc, d_conf, d_coef, d_priors, dws, d_box, d_coef_out, d_cls, d_score, d_count,
                (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_postprocess(yb_handle* h, const float* d_proto, int ph, int pw, int k, const float* d_coef, const float* d_box,
                   int n, int out_h, int out_w, int crop_masks, int mask_format, void* d_masks, int64_t* d_boxes_px,
                   float* d_proto_masks, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_proto && d_coef && d_box, "yb_postprocess: null argument");
  YB_REQUIRE(n >= 0, "yb_postprocess: negative detection count");
  if (n == 0) return YB_OK;
  CallGuard g(h);
  const PostSrc src = dense_post_src({d_proto, d_coef, d_box, d_masks, d_boxes_px, d_proto_masks, n, out_h, out_w}, ph,
                                     pw, k, mask_format);
  launch_mask_assembly(src, &src.base, 1, ph, pw, k, crop_masks, mask_format, (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_postprocess_batch(yb_handle* h, const float* d_proto, int ph, int pw, int k, const float* d_coef,
                         const float* d_box, int n, int batch, int out_h, int out_w, int crop_masks, int mask_format,
                         void* d_masks, int64_t* d_boxes_px, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_proto && d_coef && d_box, "yb_postprocess_batch: null argument");
  YB_REQUIRE(n >= 0 && batch >= 0, "yb_postprocess_batch: negative count");
  if (n == 0 || batch == 0) return YB_OK;
  CallGuard g(h);
  const PostSrc src =
      dense_post_src({d_proto, d_coef, d_box, d_masks, d_boxes_px, nullptr, n, out_h, out_w}, ph, pw, k, mask_format);
  launch_mask_assembly(src, &src.base, batch, ph, pw, k, crop_masks, mask_format, (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_postprocess_list(yb_handle* h, const yb_post_item* h_items, int B, int ph, int pw, int k, int crop_masks,
                        int mask_format, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && B >= 0 && (B == 0 || h_items), "yb_postprocess_list: bad argument");
  check_post_items(h, h_items, B, "yb_postprocess_list", true);
  if (B == 0) return YB_OK;
  YB_REQUIRE(mask_format == YB_MASK_F32 || mask_format == YB_MASK_U8 || mask_format == YB_MASK_BITS,
             "mask_assembly: unknown mask format");
  CallGuard g(h, (cudaStream_t)stream);   // shared item table: ordered behind the previous call
  PostSrc src{};
  src.table = stage_items(h->post_table, (size_t)B * sizeof(yb_post_item), h_items, B, stream);
  launch_mask_assembly(src, h_items, B, ph, pw, k, crop_masks, mask_format, (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_coco_rle_list(yb_handle* h, const yb_post_item* h_items, int B, int ph, int pw, int k, int crop_masks,
                     uint32_t* d_runs, int64_t runs_cap, char* d_chars, int64_t chars_cap, int64_t* d_row_off,
                     int32_t* d_row_len, int64_t* d_need, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && B >= 0 && (B == 0 || h_items), "yb_coco_rle_list: bad argument");
  YB_REQUIRE(d_runs && d_chars && d_row_off && d_row_len && d_need, "yb_coco_rle_list: null output");
  YB_REQUIRE(runs_cap >= 0 && chars_cap >= 0, "yb_coco_rle_list: negative capacity");
  auto on_device = [h](const void* p) { return on_handle_device(h, p); };
  YB_REQUIRE(on_device(d_runs) && on_device(d_chars) && on_device(d_row_off) && on_device(d_row_len) &&
                 on_device(d_need),
             "yb_coco_rle_list: an output is not device memory of the handle's device");
  check_post_items(h, h_items, B, "yb_coco_rle_list", false);
  CallGuard g(h, (cudaStream_t)stream);   // shared item table: ordered behind the previous call
  const yb_post_item* table =
      stage_items(h->post_table, (size_t)std::max(B, 1) * sizeof(yb_post_item), h_items, B, stream);
  launch_coco_rle(table, h_items, B, ph, pw, k, crop_masks, d_runs, runs_cap, d_chars, chars_cap, d_row_off, d_row_len,
                  d_need, (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_render_list_ex(yb_handle* h, const yb_render_item* h_items, int B, int frame_is_u8, int ph, int pw, int k,
                      int crop_masks, int top_k, float score_threshold, int class_color, float mask_alpha,
                      const float* d_palette, int P, const yb_render_opts* opts, void* stream) {
  YB_API_BEGIN
  yb_render_opts o{nullptr, 0, 0, 1};
  if (opts) o = *opts;
  YB_REQUIRE(h && B >= 0 && (B == 0 || h_items), "yb_render_list: bad argument");
  YB_REQUIRE(top_k >= 1, "yb_render_list: top_k must be >= 1");
  YB_REQUIRE(P >= 1 && d_palette, "yb_render_list: the palette needs at least one colour");
  YB_REQUIRE(on_handle_device(h, d_palette), "yb_render_list: the palette is not device memory of the handle's device");
  YB_REQUIRE(o.fps_w >= 0 && o.fps_h >= 0, "yb_render_list_ex: fps_w and fps_h must be >= 0");
  YB_REQUIRE(on_handle_device(h, o.d_counts), "yb_render_list_ex: d_counts is not device memory of the handle's device");
  auto on_device = [h](const void* p) { return on_handle_device(h, p); };
  for (int b = 0; b < B; ++b) {
    const yb_render_item& it = h_items[b];
    YB_REQUIRE(it.frame && it.out, "yb_render_list: null frame or out");
    YB_REQUIRE(it.n >= 0 && it.h > 0 && it.w > 0, "yb_render_list: n must be >= 0 and h, w > 0");
    YB_REQUIRE(it.n == 0 || (it.box && it.cls && it.score && it.det_score && (!it.proto || it.coef)),
               "yb_render_list: null coef, box, cls, score or det_score");
    YB_REQUIRE(on_device(it.frame) && on_device(it.out) && on_device(it.proto) && on_device(it.coef) &&
                   on_device(it.box) && on_device(it.cls) && on_device(it.score) && on_device(it.det_score) &&
                   on_device(it.sel_n) && on_device(it.sel_cls) && on_device(it.sel_score) && on_device(it.sel_box),
               "yb_render_list: a pointer is not device memory of the handle's device");
  }
  if (B == 0) return YB_OK;
  CallGuard g(h, (cudaStream_t)stream);   // shared item and work tables: ordered behind the previous call
  const size_t items_bytes = ((size_t)B * sizeof(yb_render_item) + 255) / 256 * 256;
  yb_render_item* table = stage_items(h->render_ws, items_bytes + render_work_bytes(B, top_k), h_items, B, stream);
  launch_render(table, h_items, B, frame_is_u8, ph, pw, k, crop_masks, top_k, score_threshold, class_color, mask_alpha,
                d_palette, P, o, reinterpret_cast<char*>(table) + items_bytes, (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_render_list(yb_handle* h, const yb_render_item* h_items, int B, int frame_is_u8, int ph, int pw, int k,
                   int crop_masks, int top_k, float score_threshold, int class_color, float mask_alpha,
                   const float* d_palette, int P, void* stream) {
  return yb_render_list_ex(h, h_items, B, frame_is_u8, ph, pw, k, crop_masks, top_k, score_threshold, class_color,
                           mask_alpha, d_palette, P, nullptr, stream);
}

int yb_maskiou(yb_handle* h, const float* d_proto_masks, int n, int ph, int pw, const int64_t* d_cls,
               float* d_maskiou, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_proto_masks && d_maskiou, "yb_maskiou: null argument");
  YB_REQUIRE(h->cfg.use_maskiou && h->finalized, "yb_maskiou: network has no maskiou_net / weights not finalized");
  if (n <= 0) return YB_OK;
  CallGuard g(h, (cudaStream_t)stream);   // shared workspaces: ordered behind the previous call
  cudaStream_t s = (cudaStream_t)stream;
  // FastMaskIoUNet (yolact.py:363-375, config.py:785-789): 5x (3x3 s2 p0 + ReLU), 1x1 + ReLU, global max.  A mask
  // needs 63 pixels on each axis (nn.Conv2d refuses anything smaller: the fifth conv would get fewer than 3 rows).
  const char* idx[6] = {"0", "2", "4", "6", "8", "10"};
  int H = ph, W = pw, C = 1;
  size_t need = 0;
  {
    int hh = ph, ww = pw;
    for (int i = 0; i < 6; ++i) {
      ConvW& cw = h->convs[std::string("maskiou_net.maskiou_net.") + idx[i]];
      int k = cw.KH, st = (i < 5) ? 2 : 1;
      hh = conv_out(hh, k, st, 0);
      ww = conv_out(ww, k, st, 0);
      YB_REQUIRE(hh >= 1 && ww >= 1, "yb_maskiou: mask too small for the network (63 x 63 at least)");
      need = std::max(need, (size_t)n * hh * ww * cw.Cout * 4);
    }
  }
  const size_t half = (need + 255) / 256 * 256;
  char* scratch = (char*)h->scratch.get(2 * half);
  const float* cur = d_proto_masks;
  for (int i = 0; i < 6; ++i) {
    ConvW& cw = h->convs[std::string("maskiou_net.maskiou_net.") + idx[i]];
    YB_REQUIRE(cw.w_f32 && cw.Cin == C, "yb_maskiou: weights missing");
    ConvProblem p;
    p.B = n;
    p.H = H;
    p.W = W;
    p.Cin = C;
    p.KH = cw.KH;
    p.KW = cw.KW;
    p.stride = (i < 5) ? 2 : 1;
    p.pad = 0;
    p.Ho = conv_out(H, cw.KH, p.stride, 0);
    p.Wo = conv_out(W, cw.KW, p.stride, 0);
    YB_REQUIRE(p.Ho >= 1 && p.Wo >= 1, "yb_maskiou: mask too small for the network");
    p.Cout = cw.Cout;
    p.act = ACT_RELU;
    p.x = cur;
    float* out = (float*)(scratch + (i & 1) * half);
    p.y = out;
    p.y_f32 = 1;
    p.y_batch_stride = (int64_t)p.Ho * p.Wo * cw.Cout;
    p.y_pix_stride = cw.Cout;
    p.bias = cw.bias;
    launch_simt_conv(p, cw.w_f32, SIMT_F32, s, &h->lc);
    cur = out;
    H = p.Ho;
    W = p.Wo;
    C = cw.Cout;
  }
  launch_maxpool_gather(cur, n, H, W, C, d_cls, d_maskiou, s, &h->lc);
  YB_API_END
}

// ---- frame preparation / eval.py consumers -----------------------------------------------------------
int yb_fast_base_transform(yb_handle* h, const void* d_img, int img_is_u8, int B, int H, int W, int out_h, int out_w,
                           int mode, const float* h_mean_bgr, const float* h_std_bgr, float* d_out, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_img && d_out, "yb_fast_base_transform: null argument");
  YB_REQUIRE(mode >= YB_XFORM_NORMALIZE && mode <= YB_XFORM_NONE, "yb_fast_base_transform: unknown transform mode");
  CallGuard g(h);
  launch_fast_base_transform(d_img, img_is_u8, B, H, W, out_h, out_w, mode, h_mean_bgr ? h_mean_bgr : kMeans,
                             h_std_bgr ? h_std_bgr : kStd, d_out, (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_pack_mask_bits(yb_handle* h, const void* d_in, int in_format, int64_t rows, int w, uint32_t* d_bits,
                      void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && rows >= 0 && w > 0 && (rows == 0 || (d_in && d_bits)), "yb_pack_mask_bits: bad argument");
  CallGuard g(h);
  launch_pack_mask_bits(d_in, in_format, rows, w, d_bits, (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_mask_iou(yb_handle* h, const uint32_t* d_a, int n, const uint32_t* d_b, int m, int64_t words, int iscrowd,
                float* d_iou, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && n >= 0 && m >= 0 && words >= 0, "yb_mask_iou: bad argument");
  YB_REQUIRE(n == 0 || m == 0 || (d_a && d_b && d_iou), "yb_mask_iou: null argument");
  CallGuard g(h);
  launch_mask_iou_bits(d_a, n, d_b, m, words, iscrowd, d_iou, (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_box_iou(yb_handle* h, const float* d_a, int n, const float* d_b, int m, int iscrowd, float* d_iou,
               void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && n >= 0 && m >= 0, "yb_box_iou: bad argument");
  YB_REQUIRE(n == 0 || m == 0 || (d_a && d_b && d_iou), "yb_box_iou: null argument");
  CallGuard g(h);
  launch_box_iou(d_a, n, d_b, m, iscrowd, d_iou, (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_mask_rle(yb_handle* h, const void* d_masks, int mask_format, int n, int mask_h, int mask_w, uint32_t* d_counts,
                int64_t cap, int32_t* d_nruns, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && n >= 0, "yb_mask_rle: bad argument");
  YB_REQUIRE(n == 0 || (d_masks && d_counts && d_nruns), "yb_mask_rle: null argument");
  CallGuard g(h);
  launch_mask_rle(d_masks, mask_format, n, mask_h, mask_w, d_counts, cap, d_nruns, (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_eval_match(yb_handle* h, const float* d_box_iou, const float* d_mask_iou, const float* d_crowd_box_iou,
                  const float* d_crowd_mask_iou, const int64_t* d_cls, const float* d_box_score, const float* d_mask_score,
                  int n, const int32_t* d_gt_cls, int g, const int32_t* d_crowd_cls, int num_crowd,
                  const double* h_thresholds, int T, int C, float* d_rec_score, int32_t* d_rec_tag, int64_t* d_counts,
                  int32_t* d_err, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && h_thresholds && d_counts && d_err, "yb_eval_match: null argument");
  eval_check_limits(n, g, num_crowd, T, C);
  YB_REQUIRE(n == 0 || (d_cls && d_box_score && d_mask_score && d_rec_score && d_rec_tag),
             "yb_eval_match: null detection argument");
  YB_REQUIRE(n == 0 || g == 0 || (d_box_iou && d_mask_iou && d_gt_cls), "yb_eval_match: null ground-truth argument");
  YB_REQUIRE(n == 0 || num_crowd == 0 || (d_crowd_box_iou && d_crowd_mask_iou && d_crowd_cls),
             "yb_eval_match: null crowd argument");
  EvalMatchSrc src{};
  yb_eval_match_item& a = src.one;
  a.box_iou = d_box_iou;
  a.mask_iou = d_mask_iou;
  a.crowd_box_iou = d_crowd_box_iou;
  a.crowd_mask_iou = d_crowd_mask_iou;
  a.cls = d_cls;
  a.box_score = d_box_score;
  a.mask_score = d_mask_score;
  a.gt_cls = d_gt_cls;
  a.crowd_cls = d_crowd_cls;
  a.n = n;
  a.g = g;
  a.num_crowd = num_crowd;
  src.T = T;
  src.C = C;
  for (int t = 0; t < T; ++t) src.thr[t] = h_thresholds[t];
  src.rec_score = d_rec_score;
  src.rec_tag = d_rec_tag;
  src.counts = d_counts;
  src.err = d_err;
  CallGuard gd(h);
  launch_eval_match(src, &src.one, 1, (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_eval_match_list(yb_handle* h, const yb_eval_match_item* h_items, int B, const double* h_thresholds, int T, int C,
                       float* d_rec_score, int32_t* d_rec_tag, int64_t* d_counts, int32_t* d_err, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && B >= 0 && (B == 0 || h_items) && h_thresholds && d_counts && d_err,
             "yb_eval_match_list: null argument");
  eval_check_limits(0, 0, 0, T, C);
  auto on_device = [h](const void* p) { return on_handle_device(h, p); };
  YB_REQUIRE(on_device(d_rec_score) && on_device(d_rec_tag) && on_device(d_counts) && on_device(d_err),
             "yb_eval_match_list: an output is not device memory of the handle's device");
  for (int b = 0; b < B; ++b) {
    const yb_eval_match_item& it = h_items[b];
    eval_check_limits(it.n, it.g, it.num_crowd, T, C);
    YB_REQUIRE(it.rec_offset >= 0, "yb_eval_match_list: negative record offset");
    if (it.n == 0) continue;
    YB_REQUIRE(it.cls && it.box_score && it.mask_score && d_rec_score && d_rec_tag,
               "yb_eval_match_list: null detection argument");
    YB_REQUIRE(it.g == 0 || (it.box_iou && it.mask_iou && it.gt_cls), "yb_eval_match_list: null ground-truth argument");
    YB_REQUIRE(it.num_crowd == 0 || (it.crowd_box_iou && it.crowd_mask_iou && it.crowd_cls),
               "yb_eval_match_list: null crowd argument");
    YB_REQUIRE(on_device(it.box_iou) && on_device(it.mask_iou) && on_device(it.crowd_box_iou) &&
                   on_device(it.crowd_mask_iou) && on_device(it.cls) && on_device(it.box_score) &&
                   on_device(it.mask_score) && on_device(it.gt_cls) && on_device(it.crowd_cls),
               "yb_eval_match_list: a pointer is not device memory of the handle's device");
  }
  EvalMatchSrc src{};
  src.T = T;
  src.C = C;
  for (int t = 0; t < T; ++t) src.thr[t] = h_thresholds[t];
  src.rec_score = d_rec_score;
  src.rec_tag = d_rec_tag;
  src.counts = d_counts;
  src.err = d_err;
  CallGuard gd(h, (cudaStream_t)stream);   // shared item table: ordered behind the previous call
  src.table = stage_items(h->eval_match_table, (size_t)std::max(B, 1) * sizeof(yb_eval_match_item), h_items, B, stream);
  launch_eval_match(src, h_items, B, (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_eval_iou_list(yb_handle* h, const yb_eval_iou_item* h_items, int B, int ph, int pw, int k, int crop_masks,
                     void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && B >= 0 && B <= 65535 && (B == 0 || h_items), "yb_eval_iou_list: bad argument");
  auto on_device = [h](const void* p) { return on_handle_device(h, p); };
  for (int b = 0; b < B; ++b) {
    const yb_eval_iou_item& it = h_items[b];
    YB_REQUIRE(it.n >= 0 && it.n <= EVAL_MAX_DETS, "yb_eval_iou_list: n must be in [0, 1024]");
    YB_REQUIRE(it.out_h > 0 && it.out_w > 0 && (int64_t)it.out_h * it.out_w <= (1ll << 28),
               "yb_eval_iou_list: out_h, out_w must be > 0, at most 2^28 pixels");
    YB_REQUIRE(it.g_all >= 0 && it.num_crowd >= 0 && it.num_crowd <= it.g_all, "yb_eval_iou_list: num_crowd outside [0, g_all]");
    YB_REQUIRE(it.g_all - it.num_crowd <= EVAL_MAX_GT && it.num_crowd <= EVAL_MAX_GT,
               "yb_eval_iou_list: at most 1024 ground truths and 1024 crowds per image");
    const int g = it.g_all - it.num_crowd;
    if (it.n > 0) {
      YB_REQUIRE(it.proto && it.coef && it.box && it.boxes_px, "yb_eval_iou_list: null proto, coef, box or boxes_px");
      YB_REQUIRE(it.g_all == 0 || (it.gt_bits && it.gt_boxes), "yb_eval_iou_list: null ground truth");
      YB_REQUIRE(g == 0 || (it.box_iou && it.mask_iou), "yb_eval_iou_list: null box_iou or mask_iou");
      YB_REQUIRE(it.num_crowd == 0 || (it.crowd_box_iou && it.crowd_mask_iou),
                 "yb_eval_iou_list: null crowd_box_iou or crowd_mask_iou");
    }
    YB_REQUIRE(on_device(it.proto) && on_device(it.coef) && on_device(it.box) && on_device(it.boxes_px) &&
                   on_device(it.gt_bits) && on_device(it.gt_boxes) && on_device(it.box_iou) && on_device(it.mask_iou) &&
                   on_device(it.crowd_box_iou) && on_device(it.crowd_mask_iou),
               "yb_eval_iou_list: a pointer is not device memory of the handle's device");
  }
  YB_REQUIRE(k % 4 == 0 && k >= 4 && k <= 128 && ph > 0 && pw > 0,
             "yb_eval_iou_list: mask_dim must be a multiple of 4 and <= 128, ph and pw > 0");
  CallGuard gd(h, (cudaStream_t)stream);   // shared item table: ordered behind the previous call
  const yb_eval_iou_item* table =
      stage_items(h->eval_iou_table, (size_t)std::max(B, 1) * sizeof(yb_eval_iou_item), h_items, B, stream);
  launch_eval_iou(table, h_items, B, ph, pw, k, crop_masks, (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_eval_ap_workspace(int64_t num_records, int T, int C, int64_t* bytes) {
  YB_API_BEGIN
  YB_REQUIRE(bytes, "yb_eval_ap_workspace: null argument");
  *bytes = (int64_t)eval_ap_workspace_bytes(num_records, T, C);
  YB_API_END
}

int yb_eval_ap(yb_handle* h, const float* d_rec_score, const int32_t* d_rec_tag, int64_t num_records,
               const int64_t* d_counts, int T, int C, void* d_work, int64_t work_bytes, double* d_ap, uint8_t* d_nonempty,
               void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_counts && d_work && d_ap && d_nonempty, "yb_eval_ap: null argument");
  YB_REQUIRE(num_records == 0 || (d_rec_score && d_rec_tag), "yb_eval_ap: null records");
  YB_REQUIRE(work_bytes >= 0, "yb_eval_ap: bad workspace size");
  CallGuard gd(h);
  launch_eval_ap(d_rec_score, d_rec_tag, num_records, d_counts, T, C, d_work, (size_t)work_bytes, d_ap, d_nonempty,
                 (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_pack_detections(yb_handle* h, const float* d_box, const float* d_coef, const int64_t* d_cls, const float* d_score,
                       const int32_t* d_count, int B, int M, int k, float* d_rec, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_box && d_coef && d_cls && d_score && d_count && d_rec, "yb_pack_detections: null argument");
  YB_REQUIRE(B >= 0 && M >= 1 && k >= 1, "yb_pack_detections: bad sizes");
  CallGuard g(h);
  launch_pack_detections(d_box, d_coef, d_cls, d_score, d_count, B, M, k, d_rec, (cudaStream_t)stream, &h->lc);
  YB_API_END
}

int yb_display_blend(yb_handle* h, const float* d_img, int img_is_255, const void* d_masks, int mask_format, int n,
                     int img_h, int img_w, const float* d_colors, float alpha, uint8_t* d_out, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_img && d_out, "yb_display_blend: null argument");
  YB_REQUIRE(n == 0 || (d_masks && d_colors), "yb_display_blend: null masks / colors");
  CallGuard g(h);
  launch_display_blend(d_img, img_is_255, d_masks, mask_format, n, img_h, img_w, d_colors, alpha, d_out,
                       (cudaStream_t)stream, &h->lc);
  YB_API_END
}

// The one implementation behind yb_dcn_forward and yb_dcn_forward_ex; the caller has validated the arguments.
static void dcn_forward(yb_handle* h, const float* d_input, const float* d_weight, const float* d_bias,
                        const float* d_offset, const float* d_mask, float* d_output, int B, int C, int H, int W, int Co,
                        const yb_dcn_params& g, int Ho, int Wo, cudaStream_t s) {
  const int taps = g.kernel_h * g.kernel_w, dg = g.deformable_group;
  const int npl = (h->cfg.precision == YB_PREC_F16X3) ? 2 : 1;
  const int sp = npl - 1;
  const bool f16 = (h->cfg.precision != YB_PREC_F32);
  const bool tc = f16 && (C / dg) % 64 == 0;
  CallGuard cg(h);
  TempPool tp;
  float* om = (float*)tp.get((size_t)B * Ho * Wo * 3 * dg * taps * 4);
  pack_om_kernel<<<grid1d((int64_t)B * Ho * Wo * 3 * dg * taps), 256, 0, s>>>(d_offset, d_mask, om, B, Ho * Wo, dg * taps);
  YB_CHECK_LAUNCH();
  // the weights are packed on the host (op-level hook, not the hot path)
  std::vector<float> hw((size_t)Co * C * taps);
  YB_CHECK_CUDA(cudaMemcpyAsync(hw.data(), d_weight, hw.size() * 4, cudaMemcpyDeviceToHost, s));
  YB_CHECK_CUDA(cudaStreamSynchronize(s));
  if (!f16) {
    float* x = (float*)tp.get((size_t)B * H * W * C * 4);
    float* y = (float*)tp.get((size_t)B * Ho * Wo * Co * 4);
    const float* wk =
        (const float*)tp.put(pack_weights(hw.data(), Co, C, g.kernel_h, g.kernel_w, nullptr, WLayout::Simt, WFormat::F32));
    launch_nchw_f32_to_nhwc<float>(d_input, x, B, C, H, W, s, &h->lc);
    launch_dcn_simt<float>(x, om, wk, d_bias, y, B, H, W, C, Ho, Wo, Co, g, ACT_NONE, 0, s, &h->lc);
    launch_nhwc_to_nchw_f32<float>(y, d_output, B, Ho, Wo, Co, s, &h->lc);
  } else {
    // the fused tensor-core kernel needs Cout % 8 == 0 and Cout >= 8: a narrower layer runs with zero weight rows and
    // zero bias up to Cp output channels, of which the first Co are copied out
    const int Cp = tc ? std::max(8, (Co + 7) / 8 * 8) : Co;
    __half* x = (__half*)tp.get((size_t)B * H * W * C * 2 * npl);
    __half* y = (__half*)tp.get((size_t)B * Ho * Wo * Cp * 2 * npl);
    launch_nchw_f32_to_nhwc<__half>(d_input, x, B, C, H, W, s, &h->lc, sp);
    if (tc) {
      const PackedWeights pw = pack_weights(hw.data(), Co, C, g.kernel_h, g.kernel_w, nullptr, WLayout::Dcn,
                                            sp ? WFormat::Split : WFormat::F16, 0, Cp);
      const __half* wk = (const __half*)tp.put(pw);
      const float* bias = d_bias;
      if (Cp > Co && d_bias) {
        float* bp = (float*)tp.get((size_t)Cp * 4);
        YB_CHECK_CUDA(cudaMemsetAsync(bp, 0, (size_t)Cp * 4, s));
        YB_CHECK_CUDA(cudaMemcpyAsync(bp, d_bias, (size_t)Co * 4, cudaMemcpyDeviceToDevice, s));
        bias = bp;
      }
      DcnTcPlan* dp = dcn_tc_plan_create(x, om, wk, bias, y, B, H, W, C, Ho, Wo, Cp, g, ACT_NONE, 0, sp, pw.out_scale);
      try {
        launch_dcn_tc(dp, s, &h->lc);
      } catch (...) {
        dcn_tc_plan_destroy(dp);
        throw;
      }
      dcn_tc_plan_destroy(dp);
    } else {
      const __half* wk = (const __half*)tp.put(
          pack_weights(hw.data(), Co, C, g.kernel_h, g.kernel_w, nullptr, WLayout::Simt, WFormat::F16));
      launch_dcn_simt<__half>(x, om, wk, d_bias, y, B, H, W, C, Ho, Wo, Co, g, ACT_NONE, 0, s, &h->lc);
    }
    if (Cp == Co) {
      launch_nhwc_to_nchw_f32<__half>(y, d_output, B, Ho, Wo, Co, s, &h->lc, sp);
    } else {
      float* yp = (float*)tp.get((size_t)B * Cp * Ho * Wo * 4);
      launch_nhwc_to_nchw_f32<__half>(y, yp, B, Ho, Wo, Cp, s, &h->lc, sp);
      const size_t plane = (size_t)Ho * Wo * 4;   // bytes of one output channel
      YB_CHECK_CUDA(cudaMemcpy2DAsync(d_output, Co * plane, yp, Cp * plane, Co * plane, B, cudaMemcpyDeviceToDevice, s));
    }
  }
  YB_CHECK_CUDA(cudaStreamSynchronize(s));  // temporaries are freed on return
}

// Ho or Wo of yb_dcn_params' geometry along one axis, 0 when the dilated kernel does not fit
static int dcn_out(int n, int k, int stride, int pad, int dil) {
  const int64_t span = (int64_t)n + 2 * (int64_t)pad - ((int64_t)dil * (k - 1) + 1);
  return span < 0 ? 0 : (int)(span / stride + 1);
}

int yb_dcn_forward(yb_handle* h, const float* d_input, const float* d_weight, const float* d_bias,
                   const float* d_offset, const float* d_mask, float* d_output, int B, int C, int H, int W, int Co,
                   int kernel_h, int kernel_w, int stride_h, int stride_w, int pad_h, int pad_w, int dilation_h,
                   int dilation_w, int deformable_group, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_input && d_weight && d_offset && d_mask && d_output, "yb_dcn_forward: null argument");
  YB_REQUIRE(kernel_h == 3 && kernel_w == 3, "yb_dcn_forward: only 3x3 kernels (all YOLACT++ DCN layers)");
  YB_REQUIRE(stride_h == stride_w && pad_h == pad_w && dilation_h == dilation_w, "yb_dcn_forward: anisotropic params");
  YB_REQUIRE(deformable_group == 1, "yb_dcn_forward: deformable_group must be 1");
  YB_REQUIRE(C % 16 == 0, "yb_dcn_forward: C must be a multiple of 16");
  YB_REQUIRE(h->cfg.precision != YB_PREC_F16X3 || C % 64 == 0,
             "yb_dcn_forward: the split-precision mode needs C % 64 == 0");
  const yb_dcn_params g{3, 3, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, 1};
  return yb_dcn_forward_ex(h, d_input, d_weight, d_bias, d_offset, d_mask, d_output, B, C, H, W, Co, &g, stream);
  YB_API_END
}

int yb_dcn_forward_ex(yb_handle* h, const float* d_input, const float* d_weight, const float* d_bias,
                      const float* d_offset, const float* d_mask, float* d_output, int B, int C, int H, int W, int Co,
                      const yb_dcn_params* p, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_input && d_weight && d_offset && d_mask && d_output && p, "yb_dcn_forward_ex: null argument");
  const yb_dcn_params g = *p;
  YB_REQUIRE(B >= 1 && C >= 1 && H >= 1 && W >= 1 && Co >= 1, "yb_dcn_forward_ex: B, C, H, W and Co must be >= 1");
  YB_REQUIRE(g.kernel_h >= 1 && g.kernel_w >= 1 && (int64_t)g.kernel_h * g.kernel_w <= 1024,
             "yb_dcn_forward_ex: kernel_h and kernel_w must be >= 1, kernel_h * kernel_w <= 1024");
  YB_REQUIRE(g.stride_h >= 1 && g.stride_w >= 1 && g.pad_h >= 0 && g.pad_w >= 0 && g.dilation_h >= 1 &&
                 g.dilation_w >= 1,
             "yb_dcn_forward_ex: stride and dilation must be >= 1, padding >= 0");
  YB_REQUIRE(g.deformable_group >= 1 && C % g.deformable_group == 0,
             "yb_dcn_forward_ex: deformable_group must be >= 1 and divide C");
  const int cg = C / g.deformable_group;
  YB_REQUIRE(h->cfg.precision != YB_PREC_F16X3 || cg % 64 == 0,
             "yb_dcn_forward_ex: the split-precision mode needs (C / deformable_group) % 64 == 0");
  YB_REQUIRE(h->cfg.precision != YB_PREC_F16TC || cg % 16 == 0,   // tensor cores at % 64, else the CUDA-core kernel
             "yb_dcn_forward_ex: the fp16 mode needs (C / deformable_group) % 16 == 0");
  const int Ho = dcn_out(H, g.kernel_h, g.stride_h, g.pad_h, g.dilation_h);
  const int Wo = dcn_out(W, g.kernel_w, g.stride_w, g.pad_w, g.dilation_w);
  YB_REQUIRE(Ho >= 1 && Wo >= 1, "yb_dcn_forward_ex: empty output");
  dcn_forward(h, d_input, d_weight, d_bias, d_offset, d_mask, d_output, B, C, H, W, Co, g, Ho, Wo, (cudaStream_t)stream);
  YB_API_END
}

int yb_dcn_psroi_pool(yb_handle* h, const float* d_input, const float* d_rois, const float* d_trans, float* d_output,
                      float* d_count, int N, int C, int H, int W, int R, int no_trans, int num_classes,
                      float spatial_scale, int output_dim, int group_size, int pooled, int part_size,
                      int sample_per_part, float trans_std, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_input && d_rois && d_output && (no_trans || d_trans), "yb_dcn_psroi_pool: null argument");
  YB_REQUIRE(N >= 1 && H >= 1 && W >= 1 && R >= 0, "yb_dcn_psroi_pool: N, H and W must be >= 1, R >= 0");
  YB_REQUIRE(pooled >= 1 && group_size >= 1 && part_size >= 1 && sample_per_part >= 1,
             "yb_dcn_psroi_pool: pooled, group_size, part_size and sample_per_part must be >= 1");
  YB_REQUIRE(output_dim >= 1 && (int64_t)C == (int64_t)output_dim * group_size * group_size,
             "yb_dcn_psroi_pool: C must be output_dim * group_size^2");
  const int ncls = no_trans ? 1 : num_classes;
  YB_REQUIRE(ncls >= 1 && output_dim % ncls == 0, "yb_dcn_psroi_pool: num_classes must be >= 1 and divide output_dim");
  CallGuard cg(h);
  cudaStream_t s = (cudaStream_t)stream;
  if (R == 0) return YB_OK;
  // the kernel reads image rois[r, 0] (truncated, as the reference's int conversion does): checked here, before
  // anything is written
  std::vector<float> bidx((size_t)R);
  YB_CHECK_CUDA(cudaMemcpy2DAsync(bidx.data(), 4, d_rois, 5 * 4, 4, (size_t)R, cudaMemcpyDeviceToHost, s));
  YB_CHECK_CUDA(cudaStreamSynchronize(s));
  for (int r = 0; r < R; ++r)
    YB_REQUIRE(bidx[r] > -1.f && bidx[r] < (float)N,   // false for NaN
               ("yb_dcn_psroi_pool: the batch index of RoI " + std::to_string(r) + " is not in [0, N)").c_str());
  PsroiPoolArgs a;
  a.x = d_input;
  a.rois = d_rois;
  a.trans = no_trans ? nullptr : d_trans;
  a.y = d_output;
  a.count = d_count;
  a.N = N, a.C = C, a.H = H, a.W = W, a.R = R;
  a.no_trans = no_trans ? 1 : 0;
  a.num_classes = ncls;
  a.output_dim = output_dim, a.group_size = group_size, a.pooled = pooled, a.part_size = part_size;
  a.sample_per_part = sample_per_part;
  a.spatial_scale = spatial_scale, a.trans_std = trans_std;
  launch_dcn_psroi_pool(a, s, &h->lc);
  YB_API_END
}

int yb_conv2d(yb_handle* h, const float* d_x, const float* h_w, const float* h_bias, const float* d_residual,
              float* d_y, int B, int Ci, int H, int W, int Co, int kh, int kw, int stride, int pad, int act,
              int precision, int iters, float* ms, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_x && h_w && d_y, "yb_conv2d: null argument");
  YB_REQUIRE(precision >= 0 && precision <= 3,
             "yb_conv2d: precision must be 0 (f32 simt), 1 (f16 tensor cores), 2 (f16 simt), 3 (split-precision tensor cores)");
  const int sp = (precision == 3) ? 1 : 0;
  CallGuard g(h);
  cudaStream_t s = (cudaStream_t)stream;
  const int Ho = conv_out(H, kh, stride, pad), Wo = conv_out(W, kw, stride, pad);
  YB_REQUIRE(Ho >= 1 && Wo >= 1, "yb_conv2d: empty output");
  TempPool tp;
  const bool f16 = precision != 0;
  const size_t es = (f16 && !sp) ? 2 : 4;   // split: two halfs per element
  void* x = tp.get((size_t)B * H * W * Ci * es);
  void* y = tp.get((size_t)B * Ho * Wo * Co * es);
  void* res = d_residual ? tp.get((size_t)B * Ho * Wo * Co * es) : nullptr;
  float* bias = nullptr;
  if (h_bias) {
    bias = (float*)tp.get((size_t)Co * 4);
    YB_CHECK_CUDA(cudaMemcpy(bias, h_bias, (size_t)Co * 4, cudaMemcpyHostToDevice));
  }
  ConvProblem p;
  p.B = B;
  p.H = H;
  p.W = W;
  p.Cin = Ci;
  p.Ho = Ho;
  p.Wo = Wo;
  p.Cout = Co;
  p.KH = kh;
  p.KW = kw;
  p.stride = stride;
  p.pad = pad;
  p.act = act;
  p.x = x;
  p.y = y;
  p.split = sp;
  p.y_pix_stride = sp ? 2 * Co : Co;
  p.y_batch_stride = (int64_t)Ho * Wo * p.y_pix_stride;
  p.bias = bias;
  p.residual = res;
  if (!f16) {
    launch_nchw_f32_to_nhwc<float>(d_x, (float*)x, B, Ci, H, W, s, &h->lc);
    if (res) launch_nchw_f32_to_nhwc<float>(d_residual, (float*)res, B, Co, Ho, Wo, s, &h->lc);
  } else {
    launch_nchw_f32_to_nhwc<__half>(d_x, (__half*)x, B, Ci, H, W, s, &h->lc, sp);
    if (res) launch_nchw_f32_to_nhwc<__half>(d_residual, (__half*)res, B, Co, Ho, Wo, s, &h->lc, sp);
  }
  std::function<void()> run;
  TcConvPlan* plan = nullptr;
  const bool tc = precision == 1 || precision == 3;
  YB_REQUIRE(!tc || tc_conv_supported(p), "yb_conv2d: shape not supported by the tensor-core kernel (Cin % 64, taps <= 9)");
  static const WFormat kFormat[4] = {WFormat::F32, WFormat::F16, WFormat::F16, WFormat::Split};
  const PackedWeights pw = pack_weights(h_w, Co, Ci, kh, kw, nullptr, tc ? WLayout::Conv : WLayout::Simt, kFormat[precision]);
  const void* wd = tp.put(pw);
  p.out_scale = pw.out_scale;
  if (tc) {
    plan = hook_tc_plan(p, (const __half*)wd, tp, s);
    run = [&]() { launch_tc_conv(plan, s, &h->lc); };
  } else {
    run = [&]() { launch_simt_conv(p, wd, precision == 2 ? SIMT_F16 : SIMT_F32, s, &h->lc); };
  }
  try {
    run();  // warm-up + result
    if (iters > 1 || ms) {
      const int n = std::max(1, iters);
      cudaEvent_t e0, e1;
      YB_CHECK_CUDA(cudaEventCreate(&e0));
      YB_CHECK_CUDA(cudaEventCreate(&e1));
      YB_CHECK_CUDA(cudaEventRecord(e0, s));
      for (int i = 0; i < n; ++i) run();
      YB_CHECK_CUDA(cudaEventRecord(e1, s));
      YB_CHECK_CUDA(cudaEventSynchronize(e1));
      float t = 0.f;
      YB_CHECK_CUDA(cudaEventElapsedTime(&t, e0, e1));
      if (ms) *ms = t / n;
      cudaEventDestroy(e0);
      cudaEventDestroy(e1);
    }
  } catch (...) {
    if (plan) tc_conv_plan_destroy(plan);
    throw;
  }
  if (plan) tc_conv_plan_destroy(plan);
  if (!f16)
    launch_nhwc_to_nchw_f32<float>((const float*)y, d_y, B, Ho, Wo, Co, s, &h->lc);
  else
    launch_nhwc_to_nchw_f32<__half>((const __half*)y, d_y, B, Ho, Wo, Co, s, &h->lc, sp);
  YB_CHECK_CUDA(cudaStreamSynchronize(s));
  YB_API_END
}

int yb_conv2d_ex(yb_handle* h, const float* d_x, const float* h_w, const float* h_bias, const float* d_residual,
                 void* d_y, int B, int Ci, int H, int W, int Co, int kh, int kw, int stride, int pad, int act,
                 int precision, const yb_conv_opts* opts, void* stream) {
  YB_API_BEGIN
  yb_conv_opts o;
  memset(&o, 0, sizeof(o));
  if (opts) o = *opts;
  YB_REQUIRE(h && d_x && h_w && (d_y || o.nseg > 0), "yb_conv2d_ex: null argument");
  YB_REQUIRE(precision >= 0 && precision <= 3, "yb_conv2d_ex: precision must be 0, 1, 2 or 3 (as yb_conv2d's)");
  YB_REQUIRE(o.nseg >= 0 && o.nseg <= 3, "yb_conv2d_ex: nseg must be 0..3");
  const bool tc = precision == 1 || precision == 3, f16 = precision != 0;
  const int sp = (precision == 3) ? 1 : 0;
  const int CiP = std::max(Ci, o.cin_pad), CoP = std::max(Co, o.cout_pad);
  YB_REQUIRE(tc || (CoP == Co && o.nseg == 0), "yb_conv2d_ex: cout_pad and nseg need the tensor cores (precision 1 or 3)");
  YB_REQUIRE(CoP == Co || (!d_residual && !o.y_f32 && o.nseg == 0),
             "yb_conv2d_ex: cout_pad does not combine with a residual, y_f32 or nseg");
  for (int i = 0; i < o.nseg; ++i)
    YB_REQUIRE(o.seg_y[i] && o.seg_begin[i] >= (i ? o.seg_end[i - 1] : 0) && o.seg_end[i] > o.seg_begin[i] &&
                   o.seg_end[i] <= Co && o.seg_pix_stride[i] >= o.seg_end[i] - o.seg_begin[i] && o.seg_batch_stride[i] >= 0,
               "yb_conv2d_ex: the segments need outputs, ascending disjoint channel ranges within Co and strides");
  const bool y_f32 = !f16 || o.y_f32;
  const int ps = o.y_pix_stride > 0 ? o.y_pix_stride : CoP;   // fp32 output pixel stride
  YB_REQUIRE(ps == CoP || (y_f32 && ps > Co && o.nseg == 0), "yb_conv2d_ex: y_pix_stride needs an fp32 output and >= Co");
  CallGuard g(h);
  cudaStream_t s = (cudaStream_t)stream;
  const int Ho = conv_out(H, kh, stride, pad), Wo = conv_out(W, kw, stride, pad);
  YB_REQUIRE(Ho >= 1 && Wo >= 1, "yb_conv2d_ex: empty output");
  if (o.poison && o.nseg == 0)
    YB_CHECK_CUDA(cudaMemsetAsync(d_y, 0xff, (size_t)B * Ho * Wo * (y_f32 ? 4 * ps : sp ? 4 * CoP : 2 * CoP), s));
  TempPool tp;
  float* bias = nullptr;
  if (h_bias) {   // zeros for the padding channels, as the network's packer writes them
    bias = (float*)tp.get((size_t)CoP * 4);
    YB_CHECK_CUDA(cudaMemsetAsync(bias, 0, (size_t)CoP * 4, s));
    YB_CHECK_CUDA(cudaMemcpyAsync(bias, h_bias, (size_t)Co * 4, cudaMemcpyHostToDevice, s));
  }
  const WFormat fmt = sp ? WFormat::Split : f16 ? WFormat::F16 : WFormat::F32;
  if (tc && kh == kw && stem_tc_supported(kh, stride, pad, Ci, Co)) {
    YB_REQUIRE(!d_residual && !o.y_f32 && !o.res_after_act && o.nseg == 0 && CiP == Ci,
               "yb_conv2d_ex: the tensor-core stem takes no residual, y_f32, res_after_act, nseg or cin_pad");
    const PackedWeights pw = pack_weights(h_w, Co, Ci, kh, kw, nullptr, WLayout::Stem, fmt);
    StemTcPlan* plan = stem_tc_plan_create(d_x, (const __half*)tp.put(pw), bias, (__half*)d_y, B, H, W, kh, stride, pad,
                                           Co, act, sp, pw.out_scale, CoP);
    try {
      launch_stem_tc(plan, s, &h->lc);
    } catch (...) {
      stem_tc_plan_destroy(plan);
      throw;
    }
    stem_tc_plan_destroy(plan);
    YB_CHECK_CUDA(cudaStreamSynchronize(s));  // temporaries are freed on return
    return YB_OK;
  }
  const size_t es = (f16 && !sp) ? 2 : 4;   // split: two halfs per element
  void* x = tp.get((size_t)B * H * W * CiP * es);
  void* res = d_residual ? tp.get((size_t)B * Ho * Wo * Co * es) : nullptr;
  if (!f16) {
    launch_nchw_f32_to_nhwc<float>(d_x, (float*)x, B, CiP, H, W, s, &h->lc);
    if (res) launch_nchw_f32_to_nhwc<float>(d_residual, (float*)res, B, Co, Ho, Wo, s, &h->lc);
  } else {
    launch_nchw_f32_to_nhwc<__half>(d_x, (__half*)x, B, CiP, H, W, s, &h->lc, sp);
    if (res) launch_nchw_f32_to_nhwc<__half>(d_residual, (__half*)res, B, Co, Ho, Wo, s, &h->lc, sp);
  }
  ConvProblem p;
  p.B = B;
  p.H = H;
  p.W = W;
  p.Cin = CiP;
  p.Ho = Ho;
  p.Wo = Wo;
  p.Cout = CoP;
  p.KH = kh;
  p.KW = kw;
  p.stride = stride;
  p.pad = pad;
  p.act = act;
  p.x = x;
  p.split = sp;
  p.bias = bias;
  p.residual = res;
  p.res_after_act = o.res_after_act ? 1 : 0;
  p.y = d_y;
  p.y_f32 = (f16 && o.y_f32) ? 1 : 0;
  p.y_pix_stride = y_f32 ? ps : sp ? 2 * CoP : CoP;
  p.y_batch_stride = (int64_t)Ho * Wo * p.y_pix_stride;
  p.nseg = o.nseg;
  for (int i = 0; i < o.nseg; ++i) {   // as the network's fused head sets them up (engine.cu fused_head)
    p.seg_begin[i] = o.seg_begin[i];
    p.seg_end[i] = o.seg_end[i];
    p.seg_act[i] = o.seg_act[i];
    p.seg_ps[i] = o.seg_pix_stride[i];
    p.seg_bs[i] = o.seg_batch_stride[i];
    p.seg_y[i] = o.seg_y[i];
  }
  if (o.nseg > 0) {
    p.y = o.seg_y[0];
    p.y_f32 = 1;
    p.y_pix_stride = o.seg_pix_stride[0];
    p.y_batch_stride = o.seg_batch_stride[0];
  }
  // input channels beyond Ci are zeros that meet zero weights: the tensor-core packer pads its rows, the CUDA-core
  // kernel gets zero-padded OIHW weights
  std::vector<float> wpad;
  const float* w = h_w;
  if (!tc && CiP > Ci) {
    const size_t taps = (size_t)kh * kw;
    wpad.assign((size_t)Co * CiP * taps, 0.f);
    for (int c = 0; c < Co; ++c) memcpy(&wpad[(size_t)c * CiP * taps], h_w + (size_t)c * Ci * taps, Ci * taps * 4);
    w = wpad.data();
  }
  YB_REQUIRE(!tc || tc_conv_supported(p), "yb_conv2d_ex: shape not supported by the tensor-core kernel (Cin % 64, taps <= 9)");
  const PackedWeights pw = tc ? pack_weights(w, Co, Ci, kh, kw, nullptr, WLayout::Conv, fmt, CiP, CoP)
                              : pack_weights(w, Co, CiP, kh, kw, nullptr, WLayout::Simt, fmt);
  const void* wd = tp.put(pw);
  p.out_scale = pw.out_scale;
  if (tc) {
    TcConvPlan* plan = hook_tc_plan(p, (const __half*)wd, tp, s);
    try {
      launch_tc_conv(plan, s, &h->lc);
    } catch (...) {
      tc_conv_plan_destroy(plan);
      throw;
    }
    tc_conv_plan_destroy(plan);
  } else {
    launch_simt_conv(p, wd, precision == 2 ? SIMT_F16 : SIMT_F32, s, &h->lc);
  }
  YB_CHECK_CUDA(cudaStreamSynchronize(s));  // temporaries are freed on return
  YB_API_END
}

int yb_resample_ex(yb_handle* h, int op, int precision, const void* d_x, const void* d_add, void* d_y, int B, int H,
                   int W, int C, int Ho, int Wo, int relu, void* stream) {
  YB_API_BEGIN
  YB_REQUIRE(h && d_x && d_y, "yb_resample_ex: null argument");
  YB_REQUIRE(op == YB_RESAMPLE_MAXPOOL || op == YB_RESAMPLE_BILINEAR, "yb_resample_ex: unknown op");
  YB_REQUIRE(precision == 0 || precision == 1 || precision == 3, "yb_resample_ex: precision must be 0, 1 or 3");
  YB_REQUIRE(B >= 1 && H >= 1 && W >= 1 && C >= 1 && Ho >= 1 && Wo >= 1, "yb_resample_ex: empty shape");
  YB_REQUIRE(C % (precision == 0 ? 4 : 8) == 0, "yb_resample_ex: C must be a multiple of the vector width (4 fp32, 8 fp16)");
  auto aligned = [](const void* p) { return ((uintptr_t)p & 15) == 0; };
  YB_REQUIRE(aligned(d_x) && aligned(d_add) && aligned(d_y), "yb_resample_ex: buffers must be 16-byte aligned");
  YB_REQUIRE(on_handle_device(h, d_x) && on_handle_device(h, d_add) && on_handle_device(h, d_y),
             "yb_resample_ex: a pointer is not device memory of the handle's device");
  if (op == YB_RESAMPLE_MAXPOOL)
    YB_REQUIRE(Ho == conv_out(H, 3, 2, 1) && Wo == conv_out(W, 3, 2, 1) && !d_add && !relu,
               "yb_resample_ex: the max pool is 3x3/2 pad 1 (Ho = (H - 1) / 2 + 1) and takes no add or relu");
  CallGuard g(h, (cudaStream_t)stream);
  cudaStream_t s = (cudaStream_t)stream;
  const int sp = precision == 3 ? 1 : 0;
  if (op == YB_RESAMPLE_MAXPOOL) {
    if (precision == 0)
      launch_maxpool3x3s2<float>((const float*)d_x, (float*)d_y, B, H, W, C, Ho, Wo, s, &h->lc);
    else
      launch_maxpool3x3s2<__half>((const __half*)d_x, (__half*)d_y, B, H, W, C, Ho, Wo, s, &h->lc, sp);
  } else {
    const float sh = bilinear_scale(H, Ho), sw = bilinear_scale(W, Wo);
    if (precision == 0)
      launch_upsample_bilinear<float>((const float*)d_x, (const float*)d_add, (float*)d_y, B, H, W, C, Ho, Wo, sh, sw,
                                      relu ? 1 : 0, s, &h->lc);
    else
      launch_upsample_bilinear<__half>((const __half*)d_x, (const __half*)d_add, (__half*)d_y, B, H, W, C, Ho, Wo, sh,
                                       sw, relu ? 1 : 0, s, &h->lc, sp);
  }
  YB_API_END
}

int64_t yb_launch_count(yb_handle* h) { return h ? h->lc.n : 0; }

int yb_set_profiling(yb_handle* h, int enable) {
  YB_API_BEGIN
  YB_REQUIRE(h, "null handle");
  h->profiling = enable != 0;
  YB_API_END
}

int yb_last_forward_ms(yb_handle* h, float* total_ms, float* conv_ms) {
  YB_API_BEGIN
  YB_REQUIRE(h, "null handle");
  if (total_ms) *total_ms = h->last_total_ms;
  if (conv_ms) *conv_ms = h->last_conv_ms;
  YB_API_END
}

int yb_last_forward_profile(yb_handle* h, char* buf, int64_t cap) {
  YB_API_BEGIN
  YB_REQUIRE(h && buf && cap > 0, "yb_last_forward_profile: bad argument");
  YB_REQUIRE(h->last_exec, "yb_last_forward_profile: no forward has run");
  std::string s;
  for (auto& op : h->last_exec->ops) s += op.name + "," + std::to_string(op.last_ms) + "\n";
  if ((int64_t)s.size() + 1 > cap) s.resize((size_t)cap - 1);
  memcpy(buf, s.c_str(), s.size() + 1);
  YB_API_END
}

int yb_set_graphs(yb_handle* h, int enable) {
  YB_API_BEGIN
  YB_REQUIRE(h, "null handle");
  h->use_graphs = enable != 0;
  YB_API_END
}

int yb_debug_chain_deps(int B, int Hin, int Win, int k, int stride, int pad, int producer_flat, int m, int32_t* out) {
  YB_API_BEGIN
  yb::tc_chain_debug_deps(B, Hin, Win, k, stride, pad, producer_flat, m, out);
  YB_API_END
}

int yb_save_plans(yb_handle* h, const char* path) {
  YB_API_BEGIN
  YB_REQUIRE(h && path, "yb_save_plans: null argument");
  CallGuard g(h);
  h->save_plans(path);
  YB_API_END
}

int yb_load_plans(yb_handle* h, const char* path) {
  YB_API_BEGIN
  YB_REQUIRE(h && path, "yb_load_plans: null argument");
  CallGuard g(h);
  h->load_plans(path);
  YB_API_END
}

int yb_plan_stats(yb_handle* h, int64_t* timed, int64_t* loaded) {
  YB_API_BEGIN
  YB_REQUIRE(h, "yb_plan_stats: null handle");
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (timed) *timed = h->plans_timed;
  if (loaded) *loaded = h->plans_loaded;
  YB_API_END
}

const char* yb_build_id(void) { return yb::build_id(); }

int yb_check_plans(const char* path, const char* out_path) {
  YB_API_BEGIN
  YB_REQUIRE(path, "yb_check_plans: null path");
  const PlanFile f = parse_plan_file(read_text_file(path));
  if (out_path) write_text_file(out_path, write_plan_file(f));
  YB_API_END
}

}  // extern "C"
