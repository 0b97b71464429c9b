// Host-side engine: weight store (reference state_dict names), BatchNorm folding + repacking,
// per-input-shape executors (activation buffers, kernel plans, CUDA graph), Detect workspaces.
#pragma once
#include <array>
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
  float* w_f32 = nullptr;    // [KH*KW*Cin][Cout]           (SIMT fp32)
  __half* w_f16 = nullptr;   // [KH*KW*Cin][Cout]           (SIMT fp16)
  __half* w_tc = nullptr;    // [KH*KW][Cout][Cin]          (tensor cores), or [1][Cout][9*Cin] for DCN
  float* bias = nullptr;     // [Cout] or null
  int pack = 0;              // 0 normal, 1 DCN ([Cout][9*Cin]), 2 stem ([Cout][Kpad], OIHW order)
  // YB_PREC_F16X3: w_tc holds [..][hi(K) | lo(K)] fp16 pairs of w * 2^e (e chosen so that max |w| * 2^e < 2^15:
  // the lo parts stay normal fp16 numbers); out_scale = 2^-e is applied to the fp32 accumulator
  float out_scale = 1.f;
};

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
  void drop_detect_state();      // frees the Detect buffers and every captured yb_infer graph (Detect parameters changed)
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
  bool fuse_heads = true;   // YB_FUSE_HEADS=0: three separate head convs per level
  bool pdl = false;         // programmatic dependent launch between consecutive tensor-core convs: on in the fp16 mode (YB_PDL=0/1)
  bool stem_on_tc = true;   // YB_STEM_TC=0 falls back to the SIMT stem
  bool dcn_fused = true;    // YB_DCN_FUSED=0: separate gather kernel + fp16 column buffer + 1x1 tensor-core contraction
  int stem_wg = 0;          // YB_STEM_WG=1|2: worker threads per output pixel in the 7x7 stem; 0 = 1 in the fp16 mode, 2 in the split mode
  bool autotune = true;     // YB_AUTOTUNE=0 disables plan-time autotuning of the tensor-core tiles
  bool pair_candidates = true;    // YB_PAIR=0: the autotuner skips CTA-pair (cluster of two) plans
  bool epi2_candidates = true;    // YB_EPI2=0: the autotuner skips plans with two MMA warpgroups (384 threads)
  float last_total_ms = 0.f, last_conv_ms = 0.f;
  yb::LaunchCounter lc;
  std::map<std::string, yb::HostTensor> host;
  std::map<std::string, yb::ConvW> convs;
  std::map<std::string, std::unique_ptr<yb::Executor>> execs;
  std::vector<void*> weight_allocs;
  std::map<std::string, std::array<int, 7>> tune_cache;  // layer shape -> (BN, stages, grid, pair, MMA warpgroups, pdl-friendly, stream-K) from the autotuner
  bool sk_candidates = true;      // the autotuner times stream-K plans: on in the split mode (YB_SK=0/1)
  int chain_mode = 1;             // runs of consecutive convs as one chain launch: 0 never, 1 when timed faster, 2 always (YB_CHAIN)
  cudaStream_t tune_stream = nullptr;   // private stream of the autotuner when PDL candidates are timed
  yb::Executor* last_exec = nullptr;
  // standalone op workspaces
  void* detect_ws = nullptr;
  size_t detect_ws_bytes = 0;
  void* scratch = nullptr;   // maskiou / dcn / conv2d temporaries
  size_t scratch_bytes = 0;
  cudaStream_t cap_stream = nullptr;  // private stream used only for CUDA-graph capture
  cudaStream_t lane_streams[8] = {};  // branch streams joined into the capture (parallel graph branches)
  cudaEvent_t ev_fork = nullptr, ev_join[8] = {};
  bool multi_stream = true;           // YB_BRANCHES=0: capture a linear graph
  // call serialisation (capi.cu CallGuard): host-side mutex + device-side ordering across caller streams
  std::recursive_mutex mu;
  cudaEvent_t ev_last = nullptr;
  cudaStream_t last_stream = nullptr;
  bool has_last = false;
  cudaStream_t capture_stream();
  ~yb_handle();

  // ---- weights
  yb::ConvW& get_conv(const std::string& conv_key, const std::string& bn_key, bool want_tc, bool want_f32,
                      bool want_f16, int pack = 0, int cin_pad = 0, int cout_pad = 0);
  int peek_cout(const std::string& conv_key) const;
  yb::ConvW& get_fused_head(const std::string& head_name);
  void finalize();
  // ---- executors
  yb::Executor* get_executor(int B, int H, int W);
  void forward(const float* d_x, int B, int H, int W, float* d_loc, float* d_conf, float* d_coef, float* d_proto,
               cudaStream_t stream);
  void infer(const float* d_x, int B, int H, int W, int cross_class, int max_out, float* d_box, float* d_coef_out,
             int64_t* d_cls, float* d_score, int32_t* d_count, float* d_proto, cudaStream_t stream);
  void* get_scratch(size_t bytes);
  void* get_detect_ws(size_t bytes);
};

namespace yb {
// builds the op list for a given input shape; dry == true only resolves weights / shapes
void build_network(yb_handle* h, Executor* ex, bool dry);
void compute_level_sizes(const yb_config& cfg, int H, int W, int level_hw[5][2], int* ph, int* pw);
std::vector<float> make_priors_host(const yb_config& cfg, const int level_hw[5][2]);
void launch_multi_copy(const void* const* src, void* const* dst, const size_t* bytes, int n, cudaStream_t stream,
                       LaunchCounter* lc);
}  // namespace yb
