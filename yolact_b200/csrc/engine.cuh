// Host-side engine: weight store (reference state_dict names), BatchNorm folding + repacking,
// per-input-shape executors (activation buffers, kernel plans, CUDA graph), Detect workspaces.
#pragma once
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "kernels.cuh"

namespace yb {

struct HostTensor {
  std::vector<float> data;
  std::vector<int64_t> shape;
  int64_t numel() const {
    int64_t n = 1;
    for (auto s : shape) n *= s;
    return n;
  }
};

// One convolution's device-resident parameters (BatchNorm already folded).
struct ConvW {
  int Cin = 0, Cout = 0, KH = 0, KW = 0;
  int cout_pad = 0;          // w_tc / bias carry this many output channels (zero rows beyond Cout): a 32-channel layer
                             // then writes 64-channel pixels the next tensor-core conv can consume; 0 = Cout
  int cin_pad = 0;           // w_tc rows are padded with zeros to this many input channels (a multiple of 64) when the
                             // producer writes zero-padded pixels (Darknet: 32 -> 64); 0 = Cin
  float* w_f32 = nullptr;    // WLayout::Simt, fp32
  __half* w_tc = nullptr;    // WLayout::Conv, Dcn or Stem (tensor cores), fp16 or split pairs
  float* bias = nullptr;     // [Cout] or null
  // YB_PREC_F16X3: w_tc holds [..][hi(K) | lo(K)] fp16 pairs of w * 2^e (e chosen so that max |w| * 2^e < 2^14:
  // the lo parts stay normal fp16 numbers); out_scale = 2^-e is applied to the fp32 accumulator
  float out_scale = 1.f;
};

// Weight packing: OIHW fp32 -> the layout and element format a kernel reads (K = taps*Cin, k = tap*Cin + c):
//   Conv  [tap][CoutP][CinP]                                  (implicit-GEMM and chain kernels)
//   Dcn   [CoutP][K], row index k                             (fused tensor-core DCN)
//   Stem  [Cout][Kpad], row index c*taps + tap (OIHW order), Kpad = stem_tc_kpad(KH)   (tensor-core stem)
//   Simt  [K][Cout], row k                                    (CUDA-core conv and DCN)
// Conv, Dcn and Stem take F16 or Split, where each row of n values becomes [hi(n) | lo(n)]; Simt takes F32 or F16.
// Other combinations are rejected.  CinP = max(Cin, cin_pad), CoutP = max(Cout, cout_pad); all padding is zeros.
// co_scale (null = 1) multiplies output channel o first (folded BatchNorm).  Split: the pairs encode w * 2^e with one
// exponent e over the whole tensor (engine.cu split_exponent), and out_scale = 2^-e.  Makes no CUDA calls.
enum class WLayout { Conv, Dcn, Stem, Simt };
enum class WFormat { F32, F16, Split };
struct PackedWeights {
  std::vector<__half> h;     // F16, Split
  std::vector<float> f;      // F32
  float out_scale = 1.f;
};
PackedWeights pack_weights(const float* oihw, int Co, int Ci, int KH, int KW, const float* co_scale, WLayout layout,
                           WFormat fmt, int cin_pad = 0, int cout_pad = 0);

// NHWC activation (element type float in YB_PREC_F32, __half in YB_PREC_F16TC unless f32 is set;
// YB_PREC_F16X3: `split` -- every pixel is [hi(C) | lo(C)] halfs, value = hi + lo)
struct Act {
  void* ptr = nullptr;
  int B = 0, H = 0, W = 0, C = 0;
  bool f32 = false;
  bool split = false;
  int64_t numel() const { return (int64_t)B * H * W * C; }
};

struct Op {
  std::function<void(cudaStream_t)> fn;
  bool is_conv = false;
  std::string name;   // layer key, for yb_last_forward_profile
  int lane = 0;       // graph branch: 0 = trunk (+ protonet); 1..5 = prediction head of FPN level lane-1
  float last_ms = 0.f;
  // tensor-core convolutions keep their problem so that runs of them can be re-planned as one chain launch
  bool has_prob = false;
  ConvProblem prob;
  const __half* w_tc = nullptr;
};

struct Executor {
  int B = 0, H = 0, W = 0;
  std::vector<void*> allocs;
  std::vector<TcConvPlan*> plans;
  std::vector<StemTcPlan*> stem_plans;
  std::vector<DcnTcPlan*> dcn_plans;
  std::vector<TcChain*> chains;
  void* sk_ws[8] = {};           // stream-K workspace per graph lane (plans of one lane are stream-ordered)
  std::vector<Op> ops;           // the conv stack (yb_forward)
  size_t fork_index = 0;         // ops[fork_index..] may run on their lanes concurrently (0 = no fork)
  float* d_in = nullptr;         // NCHW fp32 copy of the input (stable address for graph replay)
  float* loc = nullptr;          // [B,P,4]
  float* conf = nullptr;         // [B,P,C] logits
  float* coef = nullptr;         // [B,P,k]
  float* proto = nullptr;        // [B,ph,pw,k]
  float* priors = nullptr;       // [P,4]
  int64_t P = 0;
  int ph = 0, pw = 0;
  int level_hw[5][2] = {};
  Act feats[9];                  // C2..C5 (0..3), P3..P7 (4..8)
  // fused Detect (yb_infer)
  void* det_ws = nullptr;
  DetectWorkspace dws;
  float* det_box = nullptr;
  float* det_coef = nullptr;
  int64_t* det_cls = nullptr;
  float* det_score = nullptr;
  int32_t* det_count = nullptr;
  int det_cap = 0;               // rows per image the det_* buffers hold: max(nms_top_k, max_num_detections)
  // graphs: one captured yb_infer graph per (nms mode + flags, max_out); the first call of a key runs eagerly
  struct InferGraph {
    cudaGraphExec_t exec = nullptr;
    int calls = 0;
  };
  cudaGraphExec_t graph_fwd = nullptr;
  std::map<int, InferGraph> infer_graphs;
  int fwd_calls = 0;
  // uint8 frame input (yb_infer_frame_list, and yb_infer_frames as a list of equally sized frames), one per transform
  // mode, mean and std.  Every image brings its own frame and size; the entry op reads them from d_frame_table (B
  // entries, uploaded before each call), so no buffer, plan or graph depends on a frame size.  The frames replace only
  // the input: the half modes run the frame-list stem in place of ops[0], f32 runs fast_base_transform into d_in
  // ahead of ops[0]; every other op, plan and chain is this executor's.
  struct FrameInput {
    Op entry;                      // the frame stem, or fast_base_transform in YB_PREC_F32
    StemTcPlan* stem = nullptr;    // the frame stem's plan (half modes; also listed in stem_plans)
    bool replaces_stem = false;    // entry runs instead of ops[0] (half modes) or before it (f32)
    std::map<int, InferGraph> graphs;   // keyed like infer_graphs
  };
  FrameRef* d_frame_table = nullptr;
  std::map<std::string, FrameInput> frame_inputs;
  void drop_detect_state();      // frees the Detect buffers and every captured yb_infer / yb_infer_frame_list graph
  ~Executor();
};

}  // namespace yb

struct yb_handle {
  yb_config cfg;
  int device = 0;
  bool ops_only = false;
  bool finalized = false;
  bool use_graphs = true;
  bool profiling = false;
  bool pdl = false;         // programmatic dependent launch between consecutive tensor-core convs: on in the fp16 mode
  float last_total_ms = 0.f, last_conv_ms = 0.f;
  yb::LaunchCounter lc;
  std::map<std::string, yb::HostTensor> host;
  std::map<std::string, yb::ConvW> convs;
  std::map<std::string, std::unique_ptr<yb::Executor>> execs;
  std::vector<void*> weight_allocs;
  std::map<std::string, yb::TcTiling> tune_cache;  // layer shape -> the autotuner's tiling
  bool sk_candidates = true;      // the autotuner times stream-K plans: on in the split mode (YB_SK=0/1)
  int chain_mode = 1;             // runs of consecutive convs as one chain launch: 0 never, 1 when timed faster, 2 always (YB_CHAIN)
  cudaStream_t tune_stream = nullptr;   // private stream of the autotuner when PDL candidates are timed
  yb::Executor* last_exec = nullptr;
  // standalone op workspaces
  void* detect_ws = nullptr;
  size_t detect_ws_bytes = 0;
  void* scratch = nullptr;   // maskiou / dcn / conv2d temporaries
  size_t scratch_bytes = 0;
  yb_post_item* post_table = nullptr;   // yb_postprocess_list's device item table
  int post_table_cap = 0;
  void* render_ws = nullptr;            // yb_render_list's device item table and work table
  size_t render_ws_bytes = 0;
  cudaStream_t cap_stream = nullptr;  // private stream used only for CUDA-graph capture
  cudaStream_t lane_streams[8] = {};  // branch streams joined into the capture (parallel graph branches)
  cudaEvent_t ev_fork = nullptr, ev_join[8] = {};
  // call serialisation (capi.cu CallGuard): host-side mutex + device-side ordering across caller streams
  std::recursive_mutex mu;
  cudaEvent_t ev_last = nullptr;
  cudaStream_t last_stream = nullptr;
  bool has_last = false;
  cudaStream_t capture_stream();
  ~yb_handle();

  // ---- weights
  yb::ConvW& get_conv(const std::string& conv_key, const std::string& bn_key, bool want_tc, bool want_f32,
                      yb::WLayout tc_layout = yb::WLayout::Conv, int cin_pad = 0, int cout_pad = 0);
  int peek_cout(const std::string& conv_key) const;
  yb::ConvW& get_fused_head(const std::string& head_name);
  void finalize();
  // ---- executors
  yb::Executor* get_executor(int B, int H, int W);
  void forward(const float* d_x, int B, int H, int W, float* d_loc, float* d_conf, float* d_coef, float* d_proto,
               cudaStream_t stream);
  void infer(const float* d_x, int B, int H, int W, int cross_class, int max_out, float* d_box, float* d_coef_out,
             int64_t* d_cls, float* d_score, int32_t* d_count, float* d_proto, cudaStream_t stream);
  // infer on a list of B uint8 BGR frames of any sizes: frames[b] is a device [hw[2b], hw[2b+1], 3] frame, read in place
  // and FastBaseTransform'ed to H x W on the way in (same executor as infer(B,H,W))
  void infer_frame_list(const uint8_t* const* frames, const int32_t* hw, int B, int H, int W, int mode,
                        const float* mean_bgr, const float* std_bgr, int cross_class, int max_out, float* d_box,
                        float* d_coef_out, int64_t* d_cls, float* d_score, int32_t* d_count, float* d_proto,
                        cudaStream_t stream);
  void infer_on(yb::Executor* ex, yb::Executor::FrameInput* fin, const void* d_x, int cross_class, int max_out,
                float* d_box, float* d_coef_out, int64_t* d_cls, float* d_score, int32_t* d_count, float* d_proto,
                cudaStream_t stream);
  void* get_scratch(size_t bytes);
  void* get_detect_ws(size_t bytes);
  yb_post_item* get_post_table(int entries);
  void* get_render_ws(size_t bytes);
};

namespace yb {
// builds the op list for a given input shape; dry == true only resolves weights / shapes
void build_network(yb_handle* h, Executor* ex, bool dry);
void compute_level_sizes(const yb_config& cfg, int H, int W, int level_hw[5][2], int* ph, int* pw);
std::vector<float> make_priors_host(const yb_config& cfg, const int level_hw[5][2]);
void launch_multi_copy(const void* const* src, void* const* dst, const size_t* bytes, int n, cudaStream_t stream,
                       LaunchCounter* lc);
}  // namespace yb
