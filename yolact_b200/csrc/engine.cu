// Engine: see engine.cuh.  Topology follows the reference graph (file:line cited per block);
// the execution plan (NHWC, fused epilogues, direct writes into the concatenated head tensors,
// CUDA graph replay) is this repo's own.
#include "engine.cuh"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <set>

namespace yb {

// ---------------------------------------------------------------------------------------------
// small utilities
// ---------------------------------------------------------------------------------------------
static void* dmalloc(std::vector<void*>& pool, size_t bytes) {
  void* p = nullptr;
  YB_CHECK_CUDA(cudaMalloc(&p, std::max<size_t>(bytes, 256)));
  pool.push_back(p);
  return p;
}

void Executor::drop_detect_state() {
  for (auto& kv : infer_graphs)
    if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
  infer_graphs.clear();
  for (auto& fi : frame_inputs) {
    for (auto& kv : fi.second.graphs)
      if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
    fi.second.graphs.clear();
  }
  void* bufs[6] = {det_ws, det_box, det_coef, det_cls, det_score, det_count};
  for (void* b : bufs) {
    if (!b) continue;
    auto it = std::find(allocs.begin(), allocs.end(), b);
    if (it != allocs.end()) allocs.erase(it);
    cudaFree(b);
  }
  det_ws = nullptr;
  det_box = det_coef = det_score = nullptr;
  det_cls = nullptr;
  det_count = nullptr;
  det_cap = 0;
}

Executor::~Executor() {
  if (graph_fwd) cudaGraphExecDestroy(graph_fwd);
  for (auto& kv : infer_graphs)
    if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
  for (auto& fi : frame_inputs)
    for (auto& kv : fi.second.graphs)
      if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
  for (auto* c : chains) tc_chain_destroy(c);
  for (auto* p : plans) tc_conv_plan_destroy(p);
  for (auto* p : stem_plans) stem_tc_plan_destroy(p);
  for (auto* p : dcn_plans) dcn_tc_plan_destroy(p);
  for (void* p : allocs) cudaFree(p);
}

struct CopySegs {
  const void* src[8];
  void* dst[8];
  unsigned long long bytes[8];
  int n;
};
__global__ void multi_copy_kernel(CopySegs s) {
  const int seg = blockIdx.y;
  if (seg >= s.n) return;
  const unsigned long long nb = s.bytes[seg];
  const char* src = (const char*)s.src[seg];
  char* dst = (char*)s.dst[seg];
  const bool al = ((((uintptr_t)src) | ((uintptr_t)dst) | nb) & 15) == 0;
  if (al) {
    const uint4* s4 = (const uint4*)src;
    uint4* d4 = (uint4*)dst;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < nb / 16;
         i += (unsigned long long)gridDim.x * blockDim.x)
      d4[i] = s4[i];
  } else {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < nb;
         i += (unsigned long long)gridDim.x * blockDim.x)
      dst[i] = src[i];
  }
}
void launch_multi_copy(const void* const* src, void* const* dst, const size_t* bytes, int n, cudaStream_t stream,
                       LaunchCounter* lc) {
  CopySegs s;
  s.n = 0;
  size_t mx = 0;
  for (int i = 0; i < n && s.n < 8; ++i) {
    if (!dst[i] || !src[i] || bytes[i] == 0) continue;
    s.src[s.n] = src[i];
    s.dst[s.n] = dst[i];
    s.bytes[s.n] = bytes[i];
    mx = std::max(mx, bytes[i]);
    s.n++;
  }
  if (s.n == 0) return;
  int gx = (int)std::min<size_t>(132 * 8, (mx / 16 + 255) / 256 + 1);
  multi_copy_kernel<<<dim3(gx, s.n), 256, 0, stream>>>(s);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

// ---------------------------------------------------------------------------------------------
// feature-map sizes and priors (PredictionModule.make_priors, yolact.py:214-263)
// ---------------------------------------------------------------------------------------------
void compute_level_sizes(const yb_config& cfg, int H, int W, int level_hw[5][2], int* ph, int* pw) {
  int hs[8], ws[8];
  int n = 0;
  if (cfg.backbone == YB_BACKBONE_RESNET) {
    int h = conv_out(H, 7, 2, 3), w = conv_out(W, 7, 2, 3);  // stem (backbone.py:77)
    h = conv_out(h, 3, 2, 1);                                 // maxpool (backbone.py:80)
    w = conv_out(w, 3, 2, 1);
    for (int i = 0; i < cfg.num_stages; ++i) {
      if (i > 0) {
        h = conv_out(h, 3, 2, 1);
        w = conv_out(w, 3, 2, 1);
      }
      hs[n] = h;
      ws[n] = w;
      n++;
    }
  } else {
    int h = H, w = W;  // _preconv 3x3 p1 (backbone.py:267)
    for (int i = 0; i < cfg.num_stages; ++i) {
      h = conv_out(h, 3, 2, 1);
      w = conv_out(w, 3, 2, 1);
      hs[n] = h;
      ws[n] = w;
      n++;
    }
  }
  for (int l = 0; l < 3; ++l) {
    level_hw[l][0] = hs[cfg.selected_layers[l]];
    level_hw[l][1] = ws[cfg.selected_layers[l]];
  }
  for (int l = 3; l < 5; ++l) {  // FPN downsample layers 3x3 s2 p1 (yolact.py:298-302)
    level_hw[l][0] = conv_out(level_hw[l - 1][0], 3, 2, 1);
    level_hw[l][1] = conv_out(level_hw[l - 1][1], 3, 2, 1);
  }
  if (ph) *ph = level_hw[0][0] * 2;  // protonet bilinear x2 (config.py:691)
  if (pw) *pw = level_hw[0][1] * 2;
}

std::vector<float> make_priors_host(const yb_config& cfg, const int level_hw[5][2]) {
  // yolact.py:224-246: for j,i over the map; for ars in aspect_ratios (one list); for scale; for ar
  // Python evaluates in double and torch.Tensor() rounds to fp32 at the end.
  std::vector<float> out;
  for (int l = 0; l < 5; ++l) {
    const int ch = level_hw[l][0], cw = level_hw[l][1];
    for (int j = 0; j < ch; ++j)
      for (int i = 0; i < cw; ++i) {
        const double x = (i + 0.5) / cw;
        const double y = (j + 0.5) / ch;
        for (int s = 0; s < cfg.num_scales; ++s)
          for (int a = 0; a < cfg.num_ars; ++a) {
            const double scale = cfg.scales_f64[l][s] != 0.0 ? cfg.scales_f64[l][s] : (double)cfg.scales[l][s];
            const double ar = sqrt(cfg.ars_f64[a] != 0.0 ? cfg.ars_f64[a] : (double)cfg.ars[a]);  // preapply_sqrt == False
            const double w = scale * ar / cfg.max_size;  // use_pixel_scales
            double hgt = scale / ar / cfg.max_size;
            if (cfg.use_square_anchors) hgt = w;
            out.push_back((float)x);
            out.push_back((float)y);
            out.push_back((float)w);
            out.push_back((float)hgt);
          }
      }
  }
  return out;
}

// ---------------------------------------------------------------------------------------------
// network builder
// ---------------------------------------------------------------------------------------------
struct NetBuilder {
  yb_handle* h;
  Executor* ex;
  bool dry;
  bool f16;     // fp16 storage + tensor-core kernels (YB_PREC_F16TC and YB_PREC_F16X3)
  bool split;   // YB_PREC_F16X3: split-precision activations / weights, three MMA passes
  int lane = 0;
  void push(Op& op) {
    op.lane = lane;
    ex->ops.push_back(op);
  }

  size_t esize(const Act& a) const { return a.f32 ? 4 : (f16 ? 2 : 4); }

  Act alloc_act(int B, int H, int W, int C, bool f32 = false) {
    Act a;
    a.B = B;
    a.H = H;
    a.W = W;
    a.C = C;
    a.f32 = f32 || !f16;
    a.split = split && !a.f32;
    if (!dry) a.ptr = dmalloc(ex->allocs, (size_t)a.numel() * ((a.f32 || a.split) ? 4 : 2));
    return a;
  }

  struct OutSpec {       // write into an existing fp32 buffer (concatenated head outputs)
    float* base = nullptr;
    int64_t batch_stride = 0;
    int pix_stride = 0;
  };

  // conv (+ folded BN) (+ residual) (+ activation)
  Act conv(const std::string& key, const std::string& bn, const Act& in, int k, int stride, int pad, int act,
           const Act* residual = nullptr, bool out_f32 = false, const OutSpec* ospec = nullptr,
           bool in_nchw = false, bool res_after_act = false) {
    ConvProblem p;
    p.B = in.B;
    p.H = in.H;
    p.W = in.W;
    p.Cin = in.C;
    p.KH = p.KW = k;
    p.stride = stride;
    p.pad = pad;
    p.act = act;
    p.res_after_act = res_after_act ? 1 : 0;
    p.Ho = conv_out(in.H, k, stride, pad);
    p.Wo = conv_out(in.W, k, stride, pad);
    p.x = in.ptr;
    p.x_nchw_f32 = in_nchw ? 1 : 0;
    p.split = in.split ? 1 : 0;
    // the half-precision modes run every conv on the tensor cores: the network's NCHW input through the stem kernel,
    // the rest through the implicit-GEMM kernel
    const bool stem_tc = f16 && in_nchw;
    const bool tc = f16 && !in_nchw;
    YB_REQUIRE(!stem_tc || (!ospec && !out_f32 && !residual && stem_tc_supported(k, stride, pad, in.C, h->peek_cout(key))),
               ("conv " + key + ": stem shape not supported by the tensor-core stem").c_str());
    // in.C may be a zero-padded channel count (the tensor-core stem pads a 32-channel output to 64, see stem_tc)
    YB_REQUIRE(!tc || (in.C % 64 == 0 && !in.f32),
               ("conv " + key + ": the half-precision modes need fp16 inputs with Cin % 64 == 0").c_str());
    ConvW& w = stem_tc ? h->get_conv(key, bn, /*want_tc=*/true, false, WLayout::Stem)
                       : h->get_conv(key, bn, /*want_tc=*/tc, /*want_f32=*/!tc, WLayout::Conv,
                                     /*cin_pad=*/tc ? in.C : 0,
                                     // a half-precision output narrower than 64 channels (Darknet's first block: 32)
                                     // is written as zero-padded 64-channel pixels for the tensor-core conv that follows
                                     /*cout_pad=*/(tc && !out_f32 && !ospec && !residual) ? ((h->peek_cout(key) + 63) / 64) * 64 : 0);
    YB_REQUIRE((w.Cin == in.C || (tc && w.cin_pad == in.C)) && w.KH == k && w.KW == k,
               ("conv " + key + ": weight shape mismatch").c_str());
    const int cout_eff = (tc && w.cout_pad > w.Cout) ? w.cout_pad : w.Cout;   // incl. zero padding channels
    p.Cout = cout_eff;
    p.bias = w.bias;
    p.out_scale = w.out_scale;
    Act out;
    if (ospec) {
      out.B = in.B;
      out.H = p.Ho;
      out.W = p.Wo;
      out.C = w.Cout;
      out.f32 = true;
      out.ptr = ospec->base;
      p.y = ospec->base;
      p.y_f32 = 1;
      p.y_batch_stride = ospec->batch_stride;
      p.y_pix_stride = ospec->pix_stride;
    } else {
      // the tensor-core stem zero-pads its pixels to a multiple of 64 channels for the tensor-core conv that follows
      const int out_c = stem_tc ? ((w.Cout + 63) / 64) * 64 : cout_eff;
      out = alloc_act(in.B, p.Ho, p.Wo, out_c, out_f32);
      p.y = out.ptr;
      p.y_f32 = (f16 && out.f32) ? 1 : 0;
      const int ps = out.split ? 2 * cout_eff : cout_eff;
      p.y_batch_stride = (int64_t)p.Ho * p.Wo * ps;
      p.y_pix_stride = ps;
    }
    if (residual) {
      YB_REQUIRE(residual->H == p.Ho && residual->W == p.Wo && residual->C == w.Cout && residual->f32 == !f16 &&
                     residual->split == split,
                 ("conv " + key + ": residual shape mismatch").c_str());
      p.residual = residual->ptr;
    }
    if (dry) return out;
    LaunchCounter* lc = &h->lc;
    Op op;
    op.is_conv = true;
    op.name = key + " " + std::to_string(in.C) + "->" + std::to_string(w.Cout) + " k" + std::to_string(k) + "s" +
              std::to_string(stride) + " " + std::to_string(p.Ho) + "x" + std::to_string(p.Wo);
    if (stem_tc) {
      // yb_infer_frame_list replaces ops[0] with the frame-list stem
      YB_REQUIRE(ex->ops.empty() && ex->stem_plans.empty(), ("conv " + key + ": the stem must be the first op").c_str());
      StemTcPlan* sp = stem_tc_plan_create((const float*)in.ptr, w.w_tc, w.bias, (__half*)out.ptr, in.B, in.H, in.W, k,
                                           stride, pad, w.Cout, act, split ? 1 : 0, w.out_scale, out.C);
      ex->stem_plans.push_back(sp);
      op.name += " stem";
      op.fn = [sp, lc](cudaStream_t s) { launch_stem_tc(sp, s, lc); };
      push(op);
      return out;
    }
    if (tc) {
      YB_REQUIRE(tc_conv_supported(p), ("conv " + key + ": not supported by the tensor-core kernel").c_str());
      TcConvPlan* plan = autotune_tc(p, w.w_tc);
      ex->plans.push_back(plan);
      op.name += " tc " + tc_tiling_str(tc_conv_plan_tiling(plan));
      tc_conv_plan_set_pdl(plan, h->pdl ? 1 : 0);
      op.fn = [plan, lc](cudaStream_t s) { launch_tc_conv(plan, s, lc); };
      op.has_prob = true;
      op.prob = p;
      op.w_tc = w.w_tc;
    } else {
      const float* wp = w.w_f32;
      op.fn = [p, wp, lc](cudaStream_t s) { launch_simt_conv(p, wp, SIMT_F32, s, lc); };
    }
    push(op);
    return out;
  }

  Act maxpool(const Act& in) {
    Act out = alloc_act(in.B, conv_out(in.H, 3, 2, 1), conv_out(in.W, 3, 2, 1), in.C);
    if (dry) return out;
    LaunchCounter* lc = &h->lc;
    Op op;
    op.name = "maxpool";
    const int sp = in.split ? 1 : 0;
    if (f16)
      op.fn = [in, out, lc, sp](cudaStream_t s) {
        launch_maxpool3x3s2<__half>((const __half*)in.ptr, (__half*)out.ptr, in.B, in.H, in.W, in.C, out.H, out.W, s, lc, sp);
      };
    else
      op.fn = [in, out, lc](cudaStream_t s) {
        launch_maxpool3x3s2<float>((const float*)in.ptr, (float*)out.ptr, in.B, in.H, in.W, in.C, out.H, out.W, s, lc);
      };
    push(op);
    return out;
  }

  // out = bilinear(in -> [Ho,Wo]) (+ add)
  Act upsample(const Act& in, int Ho, int Wo, float sh, float sw, const Act* add, int relu) {
    Act out = alloc_act(in.B, Ho, Wo, in.C);
    if (dry) return out;
    LaunchCounter* lc = &h->lc;
    const void* addp = add ? add->ptr : nullptr;
    Op op;
    op.name = "upsample " + std::to_string(Ho) + "x" + std::to_string(Wo);
    const int sp = in.split ? 1 : 0;
    if (f16)
      op.fn = [in, out, addp, sh, sw, relu, lc, sp](cudaStream_t s) {
        launch_upsample_bilinear<__half>((const __half*)in.ptr, (const __half*)addp, (__half*)out.ptr, in.B, in.H,
                                         in.W, in.C, out.H, out.W, sh, sw, relu, s, lc, sp);
      };
    else
      op.fn = [in, out, addp, sh, sw, relu, lc](cudaStream_t s) {
        launch_upsample_bilinear<float>((const float*)in.ptr, (const float*)addp, (float*)out.ptr, in.B, in.H, in.W,
                                        in.C, out.H, out.W, sh, sw, relu, s, lc);
      };
    push(op);
    return out;
  }

  // DCN block conv2 (backbone.py:21-26): offset/mask conv + modulated deformable conv + BN + ReLU
  Act dcn(const std::string& key, const std::string& bn, const Act& in, int stride) {
    // conv_offset_mask: 3x3, same stride/pad, bias, 27 channels, fp32 output (dcn_v2.py:106-124)
    Act om = conv(key + ".conv_offset_mask", "", in, 3, stride, 1, ACT_NONE, nullptr, /*out_f32=*/true);
    ConvW& w = h->get_conv(key, bn, /*want_tc=*/f16, /*want_f32=*/!f16, WLayout::Dcn);
    YB_REQUIRE(!f16 || dcn_tc_supported(in.C, w.Cout),
               ("dcn " + key + ": the half-precision modes need C % 64 == 0 and Cout % 8 == 0 (tensor-core DCN)").c_str());
    const int Ho = om.H, Wo = om.W;
    Act out = alloc_act(in.B, Ho, Wo, w.Cout);
    if (dry) return out;
    LaunchCounter* lc = &h->lc;
    if (!f16) {
      const float* wp = w.w_f32;
      const float* bias = w.bias;
      Op op;
      op.is_conv = true;
      const int Cout = w.Cout;
      op.fn = [in, om, out, wp, bias, stride, Cout, lc](cudaStream_t s) {
        launch_dcn_simt<float>((const float*)in.ptr, (const float*)om.ptr, wp, bias, (float*)out.ptr, in.B, in.H, in.W,
                               in.C, out.H, out.W, Cout, dcn_3x3(stride), ACT_RELU, 1, s, lc);
      };
      push(op);
    } else {
      // one kernel: warp-shuffled tap geometry -> bilinear samples straight into the swizzled A stage -> wgmma
      const int sp = in.split ? 1 : 0;
      DcnTcPlan* dp = dcn_tc_plan_create((const __half*)in.ptr, (const float*)om.ptr, w.w_tc, w.bias, (__half*)out.ptr, in.B,
                                         in.H, in.W, in.C, Ho, Wo, w.Cout, dcn_3x3(stride), ACT_RELU, 1, sp, w.out_scale);
      ex->dcn_plans.push_back(dp);
      Op op;
      op.is_conv = true;
      op.name = key + " dcn_fused " + std::to_string(in.C) + "->" + std::to_string(w.Cout) + " k3s" + std::to_string(stride) +
                " " + std::to_string(Ho) + "x" + std::to_string(Wo);
      op.fn = [dp, lc](cudaStream_t s) { launch_dcn_tc(dp, s, lc); };
      push(op);
    }
    return out;
  }

  void fused_head(const std::string& hn, const Act& in, float* loc, float* conf, float* coef, int64_t P, int A, int NC,
                  int MD) {
    ConvW& w = h->get_fused_head(hn);
    const int c4 = A * 4, cc = A * NC, cm = A * MD;
    YB_REQUIRE(w.Cout == c4 + cc + cm && w.Cin == in.C, "fused head: weight shape mismatch");
    if (dry) return;
    ConvProblem p;
    p.B = in.B;
    p.H = in.H;
    p.W = in.W;
    p.Cin = in.C;
    p.KH = p.KW = 3;
    p.stride = 1;
    p.pad = 1;
    p.Ho = in.H;
    p.Wo = in.W;
    p.Cout = w.Cout;
    p.x = in.ptr;
    p.y = loc;  // unused (segments)
    p.y_f32 = 1;
    p.y_batch_stride = P * 4;
    p.y_pix_stride = c4;
    p.bias = w.bias;
    p.split = in.split ? 1 : 0;
    p.out_scale = w.out_scale;
    p.nseg = 3;
    const int begins[4] = {0, c4, c4 + cc, c4 + cc + cm};
    float* bases[3] = {loc, conf, coef};
    const int64_t bs[3] = {P * 4, P * NC, P * MD};
    const int ps[3] = {c4, cc, cm};
    const int acts[3] = {ACT_NONE, ACT_NONE, ACT_TANH};  // mask_proto_coeff_activation = tanh (yolact.py:193)
    for (int i = 0; i < 3; ++i) {
      p.seg_begin[i] = begins[i];
      p.seg_end[i] = begins[i + 1];
      p.seg_y[i] = bases[i];
      p.seg_bs[i] = bs[i];
      p.seg_ps[i] = ps[i];
      p.seg_act[i] = acts[i];
    }
    TcConvPlan* plan = autotune_tc(p, w.w_tc);
    ex->plans.push_back(plan);
    tc_conv_plan_set_pdl(plan, h->pdl ? 1 : 0);
    LaunchCounter* lc = &h->lc;
    Op op;
    op.is_conv = true;
    op.name = hn + ".bbox+conf+mask " + std::to_string(in.C) + "->" + std::to_string(w.Cout) + " k3s1 " +
              std::to_string(in.H) + "x" + std::to_string(in.W) + " tc " + tc_tiling_str(tc_conv_plan_tiling(plan));
    op.fn = [plan, lc](cudaStream_t s) { launch_tc_conv(plan, s, lc); };
    push(op);
  }

  // Runs of consecutive tensor-core convolutions in ops [begin, end) of one graph lane -- the whole ResNet trunk after
  // the max-pool (backbone.py:37-57,126-139: every bottleneck incl. the stride-2 and downsample layers), the FPN's
  // prediction / downsample layers, the protonet's 3x3 stack -- are re-planned for the chain kernel (tc_conv.cu) and
  // replaced by ONE launch when that is faster than the separately tuned launches (both are timed here).  A layer of a
  // run reads tensors written by earlier layers of the run (tracked per tile inside the kernel) or by ops before the run
  // (complete before the launch).  Returns the new end of the range.
  size_t form_chains(size_t begin, size_t end) {
    if (dry || h->chain_mode == 0) return end;
    auto& ops = ex->ops;
    // the chain's own plan of an op: one tile shape family (N tile 128, or 64 for 64-channel layers); null = not chainable
    auto chain_plan = [&](const Op& op) -> TcConvPlan* {
      if (!op.has_prob) return nullptr;
      const ConvProblem& q = op.prob;
      // "same" padding only: a stride-1 layer then keeps the resolution, which the residual-dependency pruning below relies on
      if (!(q.KH == q.KW && (q.KH == 1 || q.KH == 3) && q.pad == q.KH / 2 && (q.stride == 1 || q.stride == 2) && q.Cout % 64 == 0 && !q.y_f32 &&
            q.nseg == 0 && q.y_pix_stride == (q.split ? 2 : 1) * q.Cout && q.y_batch_stride == (int64_t)q.Ho * q.Wo * q.y_pix_stride))
        return nullptr;
      TcTiling t;
      t.bn = (q.Cout % 128 == 0) ? 128 : 64;
      t.stages = 2;
      t.mma_groups = 2;
      t.chain = 1;
      TcConvPlan* pl = nullptr;
      try {
        pl = tc_conv_plan_create(q, op.w_tc, t);
      } catch (const Error&) {
        return nullptr;
      }
      if (!tc_conv_plan_chainable(pl)) {
        tc_conv_plan_destroy(pl);
        return nullptr;
      }
      return pl;
    };
    size_t i = begin;
    while (i < end) {
      std::vector<TcConvPlan*> cp;
      size_t k = i;
      while (k < end && ops[k].lane == ops[i].lane && (!ops[k].has_prob || !ops[i].has_prob || ops[k].prob.B == ops[i].prob.B)) {
        TcConvPlan* pl = chain_plan(ops[k]);
        if (!pl) break;
        cp.push_back(pl);
        ++k;
      }
      const size_t n = k - i;
      if (n < 2) {
        for (auto* pl : cp) tc_conv_plan_destroy(pl);
        i = std::max(k, i + 1);
        continue;
      }
      // who writes what: input / residual produced inside the run -> a per-tile dependency
      std::vector<int> dep_a(n, -1), dep_r(n, -1);
      for (size_t j = 0; j < n; ++j)
        for (size_t q = 0; q < j; ++q) {
          if (ops[i + q].prob.y == ops[i + j].prob.x) dep_a[j] = (int)q;
          if (ops[i + j].prob.residual && ops[i + q].prob.y == ops[i + j].prob.residual) dep_r[j] = (int)q;
        }
      // a residual written by a layer that the input chain leads back to through stride-1 layers is complete (on the
      // rows this layer needs) whenever the input is: conv3's residual, the previous block's output, via conv2 and conv1.
      // (Every link waits for producer tiles covering at least the consumer tile's own rows -- stride 1, "same" padding --
      // and a tile only completes after its own wait was satisfied, so completion propagates down the links.)
      for (size_t j = 0; j < n; ++j) {
        if (dep_r[j] < 0) continue;
        int a = (int)j;
        for (int step = 0; step < 8 && a >= 0 && ops[i + a].prob.stride == 1; ++step) {
          a = dep_a[a];
          if (a == dep_r[j]) {
            dep_r[j] = -1;
            break;
          }
        }
      }
      // the chain, timed against the separately tuned launches -- unless this run's decision is already in the handle's
      // table (a plan file, or an earlier executor of this shape).  The key is the executor shape, the run's first and
      // last layer and every layer's shape.
      std::string ckey = std::to_string(ex->B) + "x" + std::to_string(ex->H) + "x" + std::to_string(ex->W) + ":" +
                         ops[i].name.substr(0, ops[i].name.find(' ')) + ".." +
                         ops[k - 1].name.substr(0, ops[k - 1].name.find(' ')) + ":";
      for (size_t j = i; j < k; ++j) ckey += (j > i ? ";" : "") + shape_key(ops[j].prob);
      auto known = h->chain_cache.find(ckey);
      TcChain* chain = nullptr;
      bool use = false;
      if (known != h->chain_cache.end()) {
        std::vector<const TcConvPlan*> cpl(cp.begin(), cp.end());
        try {
          chain = tc_chain_create(cpl, dep_a, dep_r);
        } catch (const Error&) {
          chain = nullptr;
        }
        if (chain && !tc_chain_graph_ok(chain)) {
          tc_chain_destroy(chain);
          chain = nullptr;
        }
        use = chain && known->second.chain;
        if (known->second.loaded) ++h->plans_loaded;
      } else {
        std::vector<const TcConvPlan*> cpl(cp.begin(), cp.end());
        const auto lc_before = h->lc.n;
        cudaEvent_t e0, e1;
        YB_CHECK_CUDA(cudaEventCreate(&e0));
        YB_CHECK_CUDA(cudaEventCreate(&e1));
        auto time_it = [&](const std::function<void()>& f) {
          float ms = 0.f;
          for (int r = 0; r < 2; ++r) f();
          YB_CHECK_CUDA(cudaEventRecord(e0, 0));
          for (int r = 0; r < 5; ++r) f();
          YB_CHECK_CUDA(cudaEventRecord(e1, 0));
          YB_CHECK_CUDA(cudaEventSynchronize(e1));
          YB_CHECK_CUDA(cudaEventElapsedTime(&ms, e0, e1));
          return ms / 5.f;
        };
        float ms_chain = 1e30f;
        try {
          chain = tc_chain_create(cpl, dep_a, dep_r);
        } catch (const Error&) {
          chain = nullptr;
        }
        if (chain && !tc_chain_graph_ok(chain)) {   // cooperative launches cannot be captured here: no chains
          tc_chain_destroy(chain);
          chain = nullptr;
        }
        if (chain) {
          ms_chain = time_it([&]() { launch_tc_chain(chain, 0, nullptr); });
          if (getenv("YB_CHAIN_STATS")) tc_chain_print_stats(chain, ops[i].name.substr(0, ops[i].name.find(' ')).c_str());
        }
        if (chain) {
          const float ms_sep = time_it([&]() {
            for (size_t j = i; j < k; ++j) ops[j].fn(0);
          });
          use = (h->chain_mode == 2) || ms_chain < ms_sep;
          ++h->plans_timed;
          h->chain_cache[ckey].chain = use;
          if (getenv("YB_CHAIN_VERBOSE"))
            fprintf(stderr, "[yolact_b200] chain %s .. %s (%zu layers): chain %.3f ms, separate %.3f ms -> %s\n",
                    ops[i].name.substr(0, ops[i].name.find(' ')).c_str(), ops[k - 1].name.substr(0, ops[k - 1].name.find(' ')).c_str(), n,
                    ms_chain, ms_sep, use ? "chain" : "separate");
        }
        h->lc.n = lc_before;   // (the separate launches counted themselves)
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
      }
      if (!use) {
        if (chain) tc_chain_destroy(chain);
        for (auto* pl : cp) tc_conv_plan_destroy(pl);
        i = k;
        continue;
      }
      ex->chains.push_back(chain);
      for (auto* pl : cp) ex->plans.push_back(pl);
      Op op;
      op.is_conv = true;
      op.lane = ops[i].lane;
      op.name = "chain x" + std::to_string(n) + " [" + ops[i].name.substr(0, ops[i].name.find(' ')) + " .. " +
                ops[k - 1].name.substr(0, ops[k - 1].name.find(' ')) + "] tc BN=128/64";
      {
        double gf = 0.0;
        for (size_t j = i; j < k; ++j) {
          const ConvProblem& q = ops[j].prob;
          gf += 2.0 * q.B * q.Ho * q.Wo * (double)q.Cin * q.Cout * q.KH * q.KW / 1e9;
        }
        char buf[48];
        snprintf(buf, sizeof(buf), " gflop=%.2f", gf);
        op.name += buf;
      }
      LaunchCounter* lc = &h->lc;
      op.fn = [chain, lc](cudaStream_t s) { launch_tc_chain(chain, s, lc); };
      ops[i] = op;
      ops.erase(ops.begin() + (i + 1), ops.begin() + k);
      end -= (n - 1);
      i = i + 1;
    }
    return end;
  }

  // stream-K workspace of the current lane (allocated on first use; the flags at its end start out zero)
  void* sk_workspace() {
    void*& ws = ex->sk_ws[lane & 7];
    if (!ws) {
      ws = dmalloc(ex->allocs, tc_conv_sk_workspace_bytes());
      YB_CHECK_CUDA(cudaMemset(ws, 0, tc_conv_sk_workspace_bytes()));
    }
    return ws;
  }

  // Plan-time autotuning of the tensor-core kernel's N tile and pipeline depth: each candidate is timed on the
  // layer's real buffers (contents irrelevant) with CUDA events; the fastest plan is kept.  Small layers
  // are launch/wave-quantisation bound and large-K ones L2-bandwidth bound, so no single rule fits.
  TcConvPlan* autotune_tc(const ConvProblem& p, const __half* w) {
    // identical layer shapes (e.g. the 23 blocks of stage 3) share one decision
    const std::string tkey = shape_key(p);
    auto it = h->tune_cache.find(tkey);
    if (it != h->tune_cache.end()) {
      TcConvPlan* pl = tc_conv_plan_create(p, w, it->second.t);
      if (it->second.loaded) {
        // a plan file's tiling is obeyed exactly or not at all
        if (tc_tiling_str(tc_conv_plan_tiling(pl)) != tc_tiling_str(it->second.t)) {
          const std::string got = tc_tiling_str(tc_conv_plan_tiling(pl));
          tc_conv_plan_destroy(pl);
          throw Error(YB_ERR_INVALID, "plan file tiling " + tkey + " (" + tc_tiling_str(it->second.t) +
                                          ") does not replay on this layer: it resolves to " + got);
        }
        ++h->plans_loaded;
      }
      if (tc_conv_plan_tiling(pl).stream_k) tc_conv_plan_set_sk_workspace(pl, sk_workspace());
      return pl;
    }
    ++h->plans_timed;
    const int bns[4] = {256, 128, 64, 32};
    const int sts[3] = {0, 3, 2};
    const int grids[3] = {device_sms(), 2 * device_sms(), 1 << 30};
    TcConvPlan* best = nullptr;
    float best_ms = 1e30f;
    std::set<std::string> seen;
    cudaEvent_t e0, e1;
    YB_CHECK_CUDA(cudaEventCreate(&e0));
    YB_CHECK_CUDA(cudaEventCreate(&e1));
    // in the fp16 mode (h->pdl) every single-CTA candidate is timed with programmatic dependent launch on a private
    // stream (consecutive launches of one kernel overlap like consecutive layers do), plus "PDL-friendly" plans that
    // leave room on the SM for the next layer's CTA
    const int npdl = h->pdl ? 2 : 1;
    cudaStream_t ts = 0;
    if (h->pdl) {
      if (!h->tune_stream) YB_CHECK_CUDA(cudaStreamCreateWithFlags(&h->tune_stream, cudaStreamNonBlocking));
      ts = h->tune_stream;
      YB_CHECK_CUDA(cudaDeviceSynchronize());
    }
    const int nsk = h->sk_candidates ? 2 : 1;   // stream-K: persistent default grid only
    for (int ki = 0; ki < nsk; ++ki)
    for (int di = 0; di < npdl; ++di)
    for (int ei = 0; ei < 2; ++ei)     // two MMA warpgroups per CTA
    for (int pi = 0; pi < 2; ++pi)     // CTA pairs (clusters of two, persistent grid only)
    for (int bi = 0; bi < 4; ++bi)
      for (int si = 0; si < 3; ++si)
        for (int gi = 0; gi < (pi ? 1 : 3); ++gi) {
          if (bns[bi] > 64 && bns[bi] >= 2 * p.Cout) continue;
          if (pi && bns[bi] < 64) continue;
          if (ei && (bns[bi] < 64 || gi == 1)) continue;   // 384-thread CTAs: one per SM
          if (di && (pi || ei || gi == 1)) continue;        // PDL-friendly: single CTAs, one MMA warpgroup, <= 1 CTA/SM of its own
          if (ki && (gi != 0 || di || h->pdl)) continue;    // stream-K: one CTA (cluster) per SM (TPC), no PDL
          TcTiling want;
          want.bn = bns[bi];
          want.stages = sts[si];
          want.grid = grids[gi];
          want.pair = pi;
          want.mma_groups = ei ? 2 : 1;
          want.pdl_friendly = di;
          want.stream_k = ki;
          TcConvPlan* cand = nullptr;
          try {
            cand = tc_conv_plan_create(p, w, want);
          } catch (const Error&) {
            continue;   // this tiling does not fit in shared memory (split precision doubles every stage)
          }
          const TcTiling got = tc_conv_plan_tiling(cand);
          if ((pi && !got.pair) || (ei && got.mma_groups != 2) || (di && !got.pdl_friendly) || (ki && !got.stream_k)) {
            tc_conv_plan_destroy(cand);
            continue;
          }
          if (ki) tc_conv_plan_set_sk_workspace(cand, sk_workspace());
          if (h->pdl) tc_conv_plan_set_pdl(cand, 1);
          if (!seen.insert(tc_tiling_str(got)).second) {  // overrides were clamped to an already-timed configuration
            tc_conv_plan_destroy(cand);
            continue;
          }
          float ms = 1e30f;
          try {
            for (int i = 0; i < 3; ++i) launch_tc_conv(cand, ts, nullptr);
            YB_CHECK_CUDA(cudaEventRecord(e0, ts));
            for (int i = 0; i < 10; ++i) launch_tc_conv(cand, ts, nullptr);
            YB_CHECK_CUDA(cudaEventRecord(e1, ts));
            YB_CHECK_CUDA(cudaEventSynchronize(e1));
            YB_CHECK_CUDA(cudaEventElapsedTime(&ms, e0, e1));
          } catch (...) {
            tc_conv_plan_destroy(cand);
            if (best) tc_conv_plan_destroy(best);
            cudaEventDestroy(e0);
            cudaEventDestroy(e1);
            throw;
          }
          if (ms < best_ms) {
            if (best) tc_conv_plan_destroy(best);
            best = cand;
            best_ms = ms;
          } else {
            tc_conv_plan_destroy(cand);
          }
        }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    YB_REQUIRE(best != nullptr, "autotune: no candidate");
    h->tune_cache[tkey].t = tc_conv_plan_tiling(best);
    return best;
  }

  // the autotuner's key of a layer: every problem field a tiling's validity or speed depends on (no pointers), so
  // that layers of one shape share a decision within a handle and across processes (plan files)
  static std::string shape_key(const ConvProblem& p) {
    return std::to_string(p.B) + "," + std::to_string(p.H) + "," + std::to_string(p.W) + "," + std::to_string(p.Cin) +
           "," + std::to_string(p.Cout) + "," + std::to_string(p.KH) + "," + std::to_string(p.stride) + "," +
           std::to_string(p.pad) + "," + (p.residual ? "r" : "-") + (p.y_f32 ? "f" : "h") + (p.split ? "s" : "") +
           std::to_string(p.nseg) + "," + std::to_string(p.y_pix_stride) + "," + std::to_string((long long)p.y_batch_stride);
  }
};

static bool block_uses_dcn(const yb_config& cfg, int stage, int j) {
  // backbone.py:112-118
  const int blocks = cfg.layers[stage];
  const int dl = cfg.dcn_layers[stage];
  if (j == 0) return dl >= blocks;
  const int interval = cfg.dcn_interval > 0 ? cfg.dcn_interval : 1;
  return ((j + dl) >= blocks) && (j % interval == 0);
}

void build_network(yb_handle* h, Executor* ex, bool dry) {
  const yb_config& cfg = h->cfg;
  NetBuilder nb{h, ex, dry, cfg.precision != YB_PREC_F32, cfg.precision == YB_PREC_F16X3};
  const int B = ex->B, H = ex->H, W = ex->W;
  const int NC = cfg.num_classes, MD = cfg.mask_dim, A = cfg.num_scales * cfg.num_ars;

  compute_level_sizes(cfg, H, W, ex->level_hw, &ex->ph, &ex->pw);
  ex->P = 0;
  int64_t level_off[5];
  for (int l = 0; l < 5; ++l) {
    level_off[l] = ex->P;
    ex->P += (int64_t)ex->level_hw[l][0] * ex->level_hw[l][1] * A;
  }
  if (!dry) {
    ex->d_in = (float*)dmalloc(ex->allocs, (size_t)B * 3 * H * W * 4);
    ex->loc = (float*)dmalloc(ex->allocs, (size_t)B * ex->P * 4 * 4);
    ex->conf = (float*)dmalloc(ex->allocs, (size_t)B * ex->P * NC * 4);
    ex->coef = (float*)dmalloc(ex->allocs, (size_t)B * ex->P * MD * 4);
    std::vector<float> pri = make_priors_host(cfg, ex->level_hw);
    YB_REQUIRE((int64_t)pri.size() == ex->P * 4, "prior count mismatch");
    ex->priors = (float*)dmalloc(ex->allocs, pri.size() * 4);
    YB_CHECK_CUDA(cudaMemcpy(ex->priors, pri.data(), pri.size() * 4, cudaMemcpyHostToDevice));
  }

  // ---------------- backbone ----------------
  Act in;
  in.B = B;
  in.H = H;
  in.W = W;
  in.C = 3;
  in.f32 = true;
  in.ptr = ex->d_in;
  std::vector<Act> outs;
  if (cfg.backbone == YB_BACKBONE_RESNET) {
    // backbone.py:126-139: conv1 7x7/2 + bn1 + relu + maxpool, then Bottleneck stages
    Act x = nb.conv("backbone.conv1", "backbone.bn1", in, 7, 2, 3, ACT_RELU, nullptr, false, nullptr, /*nchw*/ true);
    x = nb.maxpool(x);
    for (int i = 0; i < cfg.num_stages; ++i) {
      const int stride = (i == 0) ? 1 : 2;
      for (int j = 0; j < cfg.layers[i]; ++j) {
        const std::string n = "backbone.layers." + std::to_string(i) + "." + std::to_string(j);
        // Bottleneck.forward, backbone.py:37-57 (stride on conv2, :22,28)
        Act o = nb.conv(n + ".conv1", n + ".bn1", x, 1, 1, 0, ACT_RELU);
        const int s2 = (j == 0) ? stride : 1;
        if (block_uses_dcn(cfg, i, j))
          o = nb.dcn(n + ".conv2", n + ".bn2", o, s2);
        else
          o = nb.conv(n + ".conv2", n + ".bn2", o, 3, s2, 1, ACT_RELU);
        Act identity = x;
        if (j == 0) identity = nb.conv(n + ".downsample.0", n + ".downsample.1", x, 1, stride, 0, ACT_NONE);
        x = nb.conv(n + ".conv3", n + ".bn3", o, 1, 1, 0, ACT_RELU, &identity);
      }
      outs.push_back(x);
      if (i < 4) ex->feats[i] = x;
    }
  } else {
    // DarkNetBackbone.forward, backbone.py:299-309; conv -> BN -> LeakyReLU(0.1) (:222-233);
    // DarkNetBlock: conv2(conv1(x)) + x with no activation after the add (:235-247)
    Act x = nb.conv("backbone._preconv.0", "backbone._preconv.1", in, 3, 1, 1, ACT_LEAKY, nullptr, false, nullptr, true);
    for (int i = 0; i < cfg.num_stages; ++i) {
      const std::string ln = "backbone.layers." + std::to_string(i);
      x = nb.conv(ln + ".0.0", ln + ".0.1", x, 3, 2, 1, ACT_LEAKY);
      for (int j = 0; j < cfg.layers[i]; ++j) {
        const std::string n = ln + "." + std::to_string(j + 1);
        Act o = nb.conv(n + ".conv1.0", n + ".conv1.1", x, 1, 1, 0, ACT_LEAKY);
        // the add happens AFTER conv2's LeakyReLU and nothing follows it (backbone.py:246-247)
        x = nb.conv(n + ".conv2.0", n + ".conv2.1", o, 3, 1, 1, ACT_LEAKY, &x, false, nullptr, false, /*res_after_act=*/true);
      }
      outs.push_back(x);
      if (i < 4) ex->feats[i] = x;
    }
  }

  // ---------------- FPN (yolact.py:311-361) ----------------
  Act C[3] = {outs[cfg.selected_layers[0]], outs[cfg.selected_layers[1]], outs[cfg.selected_layers[2]]};
  // lat_layers / pred_layers are stored in reverse: index 0 <-> deepest level (yolact.py:286-289,324-341)
  Act x5 = nb.conv("fpn.lat_layers.0", "", C[2], 1, 1, 0, ACT_NONE);
  Act l4 = nb.conv("fpn.lat_layers.1", "", C[1], 1, 1, 0, ACT_NONE);
  Act x4 = nb.upsample(x5, l4.H, l4.W, bilinear_scale(x5.H, l4.H), bilinear_scale(x5.W, l4.W), &l4, 0);
  Act l3 = nb.conv("fpn.lat_layers.2", "", C[0], 1, 1, 0, ACT_NONE);
  Act x3 = nb.upsample(x4, l3.H, l3.W, bilinear_scale(x4.H, l3.H), bilinear_scale(x4.W, l3.W), &l3, 0);
  Act Pl[5];
  Pl[2] = nb.conv("fpn.pred_layers.0", "", x5, 3, 1, 1, ACT_RELU);
  Pl[1] = nb.conv("fpn.pred_layers.1", "", x4, 3, 1, 1, ACT_RELU);
  Pl[0] = nb.conv("fpn.pred_layers.2", "", x3, 3, 1, 1, ACT_RELU);
  Pl[3] = nb.conv("fpn.downsample_layers.0", "", Pl[2], 3, 2, 1, ACT_NONE);
  Pl[4] = nb.conv("fpn.downsample_layers.1", "", Pl[3], 3, 2, 1, ACT_NONE);
  for (int l = 0; l < 5; ++l) ex->feats[4 + l] = Pl[l];
  nb.form_chains(0, ex->ops.size());
  ex->fork_index = ex->ops.size();   // protonet (lane 0) and the 5 head levels (lanes 1..5) are independent

  // ---------------- protonet on P3 (config.py:691, utils/functions.py:163-213, yolact.py:588-599) ----
  {
    Act p = nb.conv("proto_net.0", "", Pl[0], 3, 1, 1, ACT_RELU);
    p = nb.conv("proto_net.2", "", p, 3, 1, 1, ACT_RELU);
    p = nb.conv("proto_net.4", "", p, 3, 1, 1, ACT_RELU);
    // InterpolateModule(scale_factor=2) + ReLU
    p = nb.upsample(p, p.H * 2, p.W * 2, bilinear_scale(p.H, p.H * 2), bilinear_scale(p.W, p.W * 2), nullptr, 1);
    p = nb.conv("proto_net.8", "", p, 3, 1, 1, ACT_RELU);
    // 1x1 -> mask_dim, then mask_proto_prototype_activation = relu (yolact.py:589); NHWC fp32 == permute(0,2,3,1)
    p = nb.conv("proto_net.10", "", p, 1, 1, 0, ACT_RELU, nullptr, /*out_f32=*/true);
    ex->proto = (float*)p.ptr;
    YB_REQUIRE(p.H == ex->ph && p.W == ex->pw && p.C == MD, "proto shape mismatch");
    nb.form_chains(ex->fork_index, ex->ops.size());   // proto_net.0 / .2 / .4: three 3x3 layers at one resolution
  }

  // ---------------- shared prediction head over the 5 levels (yolact.py:133-212, 616-634) -----------
  for (int l = 0; l < 5; ++l) {
    nb.lane = 1 + l;
    const std::string hn = "prediction_layers.0";
    Act u = nb.conv(hn + ".upfeature.0", "", Pl[l], 3, 1, 1, ACT_RELU);
    if (nb.f16) {
      // bbox + conf + mask convs share their input: one tensor-core launch with Cout = A*(4+C+k), the epilogue
      // routes channel ranges to the three concatenated fp32 tensors (tanh on the mask coefficients)
      nb.fused_head(hn, u, ex->loc ? ex->loc + level_off[l] * 4 : nullptr, ex->conf ? ex->conf + level_off[l] * NC : nullptr,
                    ex->coef ? ex->coef + level_off[l] * MD : nullptr, ex->P, A, NC, MD);
      continue;
    }
    NetBuilder::OutSpec os;
    os.base = ex->loc ? ex->loc + level_off[l] * 4 : nullptr;
    os.batch_stride = ex->P * 4;
    os.pix_stride = A * 4;
    nb.conv(hn + ".bbox_layer", "", u, 3, 1, 1, ACT_NONE, nullptr, true, &os);
    os.base = ex->conf ? ex->conf + level_off[l] * NC : nullptr;
    os.batch_stride = ex->P * NC;
    os.pix_stride = A * NC;
    nb.conv(hn + ".conf_layer", "", u, 3, 1, 1, ACT_NONE, nullptr, true, &os);
    os.base = ex->coef ? ex->coef + level_off[l] * MD : nullptr;
    os.batch_stride = ex->P * MD;
    os.pix_stride = A * MD;
    nb.conv(hn + ".mask_layer", "", u, 3, 1, 1, ACT_TANH, nullptr, true, &os);  // mask_proto_coeff_activation = tanh
  }
}

}  // namespace yb

// ---------------------------------------------------------------------------------------------
// yb_handle
// ---------------------------------------------------------------------------------------------
using namespace yb;

yb_handle::~yb_handle() {
  execs.clear();
  for (void* p : weight_allocs) cudaFree(p);
  if (cap_stream) cudaStreamDestroy(cap_stream);
  if (tune_stream) cudaStreamDestroy(tune_stream);
  for (auto s : lane_streams)
    if (s) cudaStreamDestroy(s);
  if (ev_fork) cudaEventDestroy(ev_fork);
  if (ev_last) cudaEventDestroy(ev_last);
  for (auto e : ev_join)
    if (e) cudaEventDestroy(e);
}

cudaStream_t yb_handle::capture_stream() {
  if (!cap_stream) YB_CHECK_CUDA(cudaStreamCreateWithFlags(&cap_stream, cudaStreamNonBlocking));
  return cap_stream;
}

void* yb::DeviceBuffer::get(size_t bytes) {
  if (bytes > bytes_) {
    const size_t cap = floor_ ? std::max(bytes, std::max(floor_, 2 * bytes_)) : bytes;
    if (ptr_) {
      YB_CHECK_CUDA(cudaDeviceSynchronize());
      cudaFree(ptr_);
      ptr_ = nullptr;
      bytes_ = 0;
    }
    YB_CHECK_CUDA(cudaMalloc(&ptr_, cap));
    bytes_ = cap;
  }
  return ptr_;
}

int yb_handle::peek_cout(const std::string& conv_key) const {
  auto it = host.find(conv_key + ".weight");
  return (it == host.end() || it->second.shape.empty()) ? 0 : (int)it->second.shape[0];
}

// ---- weight packing (engine.cuh pack_weights) -----------------------------------------------------------------------
// Split precision: w * 2^e = hi + lo with hi = rn_fp16(w * 2^e), lo = rn_fp16(w * 2^e - hi).  e puts the largest |w|
// of the tensor just below 2^14, so that hi never overflows and lo (<= 2^-11 |hi|) is a normal fp16 number for every
// weight larger than 2^-17 of the tensor's maximum; the kernels multiply the fp32 accumulator by 2^-e (exact).
static int split_exponent(float max_abs) {
  if (!(max_abs > 0.f) || !std::isfinite(max_abs)) return 0;
  int ex = 0;
  frexpf(max_abs, &ex);          // max_abs = m * 2^ex, m in [0.5, 1)
  return std::max(-24, std::min(40, 14 - ex));
}

PackedWeights yb::pack_weights(const float* w, int Co, int Ci, int KH, int KW, const float* co_scale, WLayout layout,
                           WFormat fmt, int cin_pad, int cout_pad) {
  const bool simt = layout == WLayout::Simt, split = fmt == WFormat::Split;
  YB_REQUIRE(simt ? !split : fmt != WFormat::F32, "pack_weights: no kernel reads this layout in this format");
  const int CiP = std::max(Ci, cin_pad), CoP = std::max(Co, cout_pad);
  YB_REQUIRE(CiP == Ci || layout == WLayout::Conv, "pack_weights: only the conv layout pads input channels");
  YB_REQUIRE(CoP == Co || layout == WLayout::Conv || layout == WLayout::Dcn,
             "pack_weights: only the conv and DCN layouts pad output channels");
  const int taps = KH * KW;
  const size_t K = (size_t)taps * Ci;
  auto value = [&](int o, size_t i) { return co_scale ? w[o * K + i] * co_scale[o] : w[o * K + i]; };   // i = c*taps + t
  PackedWeights pw;
  if (simt) {   // [tap*Cin + c][Cout]
    if (fmt == WFormat::F32) pw.f.resize(K * Co);
    else pw.h.resize(K * Co);
    for (int o = 0; o < Co; ++o)
      for (int c = 0; c < Ci; ++c)
        for (int t = 0; t < taps; ++t) {
          const size_t d = ((size_t)t * Ci + c) * Co + o;
          const float v = value(o, (size_t)c * taps + t);
          if (fmt == WFormat::F32) pw.f[d] = v;
          else pw.h[d] = from_f32<__half>(v);
        }
    return pw;
  }
  float up = 1.f;
  if (split) {   // one power of two for the whole tensor
    float mx = 0.f;
    for (int o = 0; o < Co; ++o)
      for (size_t i = 0; i < K; ++i) mx = std::max(mx, fabsf(value(o, i)));
    const int e = split_exponent(mx);
    up = ldexpf(1.f, e);
    pw.out_scale = ldexpf(1.f, -e);
  }
  // tensor-core layouts: rows of L halfs (split: of 2*L halfs, [hi(L) | lo(L)])
  const size_t L = layout == WLayout::Conv ? (size_t)CiP : layout == WLayout::Dcn ? K : (size_t)stem_tc_kpad(KH);
  const size_t rows = layout == WLayout::Conv ? (size_t)taps * CoP : layout == WLayout::Dcn ? (size_t)CoP : (size_t)Co;
  YB_REQUIRE(layout != WLayout::Stem || K <= L, "pack_weights: too many stem input channels");
  const size_t row_len = split ? 2 * L : L;
  pw.h.assign(rows * row_len, __float2half_rn(0.f));
  for (int o = 0; o < Co; ++o)
    for (int c = 0; c < Ci; ++c)
      for (int t = 0; t < taps; ++t) {
        __half* d = layout == WLayout::Conv ? &pw.h[((size_t)t * CoP + o) * row_len + c]
                    : layout == WLayout::Dcn ? &pw.h[o * row_len + (size_t)t * Ci + c]
                                             : &pw.h[o * row_len + (size_t)c * taps + t];
        const float v = value(o, (size_t)c * taps + t);
        if (split) split_f32(v * up, d[0], d[L]);
        else d[0] = from_f32<__half>(v);
      }
  return pw;
}

template <typename T>
static T* upload(std::vector<void*>& pool, const std::vector<T>& v) {
  T* d = (T*)dmalloc(pool, v.size() * sizeof(T));
  YB_CHECK_CUDA(cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  return d;
}

static const HostTensor& need(yb_handle* h, const std::string& name) {
  auto it = h->host.find(name);
  if (it == h->host.end()) throw Error(YB_ERR_MISSING_WEIGHT, "missing weight: " + name);
  return it->second;
}

ConvW& yb_handle::get_conv(const std::string& conv_key, const std::string& bn_key, bool want_tc, bool want_f32,
                           WLayout tc_layout, int cin_pad, int cout_pad) {
  ConvW& cw = convs[conv_key];
  const HostTensor& w = need(this, conv_key + ".weight");
  YB_REQUIRE(w.shape.size() == 4, ("weight " + conv_key + " is not 4-D").c_str());
  const int Co = (int)w.shape[0], Ci = (int)w.shape[1], KH = (int)w.shape[2], KW = (int)w.shape[3];
  const bool pad = want_tc && tc_layout == WLayout::Conv;
  const int CiP = (pad && cin_pad > Ci) ? cin_pad : Ci;   // row length of the tensor-core packing
  const int CoP = (pad && cout_pad > Co) ? cout_pad : Co;  // rows of the tensor-core packing (zeros beyond Co)
  if (cw.Cout == 0) {
    cw.cout_pad = CoP;
    cw.cin_pad = CiP;
    cw.Cin = Ci;
    cw.Cout = Co;
    cw.KH = KH;
    cw.KW = KW;
  }
  const bool has_bias = host.count(conv_key + ".bias") > 0;
  const bool has_bn = !bn_key.empty();
  const bool need_f32 = want_f32 && !cw.w_f32;
  const bool need_tc = want_tc && !cw.w_tc;
  if (!need_f32 && !need_tc && (cw.bias || (!has_bias && !has_bn))) return cw;

  // fold BatchNorm (eval mode, eps = 1e-5): w' = w * g/sqrt(v+eps); b' = beta + (b - mean) * g/sqrt(v+eps)
  std::vector<float> scale(Co, 1.f), shift(Co, 0.f);
  if (has_bias) {
    const HostTensor& b = need(this, conv_key + ".bias");
    YB_REQUIRE(b.numel() == Co, ("bias " + conv_key + " has the wrong size").c_str());
    for (int o = 0; o < Co; ++o) shift[o] = b.data[o];
  }
  if (has_bn) {
    const HostTensor& g = need(this, bn_key + ".weight");
    const HostTensor& be = need(this, bn_key + ".bias");
    const HostTensor& mu = need(this, bn_key + ".running_mean");
    const HostTensor& var = need(this, bn_key + ".running_var");
    YB_REQUIRE(g.numel() == Co && be.numel() == Co && mu.numel() == Co && var.numel() == Co,
               ("batchnorm " + bn_key + " has the wrong size").c_str());
    for (int o = 0; o < Co; ++o) {
      const float s = g.data[o] / sqrtf(var.data[o] + 1e-5f);
      scale[o] = s;
      shift[o] = be.data[o] + (shift[o] - mu.data[o]) * s;
    }
  }
  if (need_f32)
    cw.w_f32 = upload(weight_allocs, pack_weights(w.data.data(), Co, Ci, KH, KW, scale.data(), WLayout::Simt, WFormat::F32).f);
  if (need_tc) {
    const WFormat fmt = cfg.precision == YB_PREC_F16X3 ? WFormat::Split : WFormat::F16;
    PackedWeights pw = pack_weights(w.data.data(), Co, Ci, KH, KW, scale.data(), tc_layout, fmt, CiP, CoP);
    cw.w_tc = upload(weight_allocs, pw.h);
    cw.out_scale = pw.out_scale;
  }
  if (!cw.bias && (has_bias || has_bn)) {
    shift.resize((size_t)std::max(Co, cw.cout_pad), 0.f);   // zero bias for the padding channels
    cw.bias = upload(weight_allocs, shift);
  }
  return cw;
}

ConvW& yb_handle::get_fused_head(const std::string& hn) {
  ConvW& cw = convs[hn + ".fused"];
  if (cw.w_tc) return cw;
  const char* parts[3] = {".bbox_layer", ".conf_layer", ".mask_layer"};
  int Ci = 0, Co = 0;
  for (int i = 0; i < 3; ++i) {
    const HostTensor& w = need(this, hn + parts[i] + ".weight");
    YB_REQUIRE(w.shape.size() == 4 && w.shape[2] == 3 && w.shape[3] == 3, "fused head: 3x3 convs expected");
    YB_REQUIRE(Ci == 0 || Ci == (int)w.shape[1], "fused head: Cin mismatch");
    Ci = (int)w.shape[1];
    Co += (int)w.shape[0];
  }
  // the three heads' OIHW weights as one conv: one power-of-two scale for all of them (they share the accumulator tile)
  std::vector<float> oihw;
  std::vector<float> bias(Co, 0.f);
  int o0 = 0;
  for (int i = 0; i < 3; ++i) {
    const HostTensor& w = need(this, hn + parts[i] + ".weight");
    oihw.insert(oihw.end(), w.data.begin(), w.data.end());
    auto it = host.find(hn + parts[i] + ".bias");
    if (it != host.end()) std::copy_n(it->second.data.begin(), w.shape[0], bias.begin() + o0);
    o0 += (int)w.shape[0];
  }
  const WFormat fmt = cfg.precision == YB_PREC_F16X3 ? WFormat::Split : WFormat::F16;
  PackedWeights pw = pack_weights(oihw.data(), Co, Ci, 3, 3, nullptr, WLayout::Conv, fmt);
  cw.Cin = Ci;
  cw.Cout = Co;
  cw.KH = cw.KW = 3;
  cw.out_scale = pw.out_scale;
  cw.w_tc = upload(weight_allocs, pw.h);
  cw.bias = upload(weight_allocs, bias);
  return cw;
}

void yb_handle::finalize() {
  YB_REQUIRE(!ops_only, "finalize: this handle was created without a network");
  execs.clear();
  last_exec = nullptr;
  // drop previously packed weights (weights may be re-loaded)
  YB_CHECK_CUDA(cudaDeviceSynchronize());
  for (void* p : weight_allocs) cudaFree(p);
  weight_allocs.clear();
  convs.clear();
  Executor dry;
  dry.B = 1;
  dry.H = cfg.max_size;
  dry.W = cfg.max_size;
  build_network(this, &dry, /*dry=*/true);
  if (cfg.use_maskiou) {
    const char* idx[6] = {"0", "2", "4", "6", "8", "10"};
    for (int i = 0; i < 6; ++i) get_conv(std::string("maskiou_net.maskiou_net.") + idx[i], "", false, true);
  }
  finalized = true;
}

Executor* yb_handle::get_executor(int B, int H, int W) {
  YB_REQUIRE(finalized, "forward called before yb_finalize_weights");
  const std::string key = std::to_string(B) + "x" + std::to_string(H) + "x" + std::to_string(W);
  auto it = execs.find(key);
  if (it != execs.end()) return it->second.get();
  std::unique_ptr<Executor> ex(new Executor());
  ex->B = B;
  ex->H = H;
  ex->W = W;
  build_network(this, ex.get(), /*dry=*/false);
  Executor* raw = ex.get();
  execs[key] = std::move(ex);
  return raw;
}

// fin (yb_infer_frame_list): its entry op runs first, in place of ops[0] when it replaces the stem
static void run_ops(yb_handle* h, Executor* ex, cudaStream_t stream, bool branches = false,
                    const Executor::FrameInput* fin = nullptr) {
  static const bool trace = getenv("YB_TRACE") != nullptr;   // debug: name every op and sync after it
  const size_t first = (fin && fin->replaces_stem) ? 1 : 0;
  if (trace) {
    auto run = [&](const Op& op) {
      fprintf(stderr, "[yb] %s ...", op.name.c_str());
      fflush(stderr);
      op.fn(stream);
      cudaError_t e = cudaStreamSynchronize(stream);
      fprintf(stderr, " %s\n", e == cudaSuccess ? "ok" : cudaGetErrorString(e));
      fflush(stderr);
    };
    if (fin) run(fin->entry);
    for (size_t i = first; i < ex->ops.size(); ++i) run(ex->ops[i]);
    return;
  }
  if (fin) fin->entry.fn(stream);
  if (!branches || ex->fork_index == 0 || ex->fork_index >= ex->ops.size()) {
    for (size_t i = first; i < ex->ops.size(); ++i) ex->ops[i].fn(stream);
    return;
  }
  // trunk, then fork: each lane gets its own stream so that the captured graph has parallel branches
  // (small latency-bound head convs fill the gaps of the large protonet convs)
  for (size_t i = first; i < ex->fork_index; ++i) ex->ops[i].fn(stream);
  if (!h->ev_fork) YB_CHECK_CUDA(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
  YB_CHECK_CUDA(cudaEventRecord(h->ev_fork, stream));
  bool used[8] = {false, false, false, false, false, false, false, false};
  for (size_t i = ex->fork_index; i < ex->ops.size(); ++i) {
    const int lane = ex->ops[i].lane & 7;
    cudaStream_t s = stream;
    if (lane > 0) {
      if (!h->lane_streams[lane]) YB_CHECK_CUDA(cudaStreamCreateWithFlags(&h->lane_streams[lane], cudaStreamNonBlocking));
      s = h->lane_streams[lane];
      if (!used[lane]) {
        YB_CHECK_CUDA(cudaStreamWaitEvent(s, h->ev_fork, 0));
        used[lane] = true;
      }
    }
    ex->ops[i].fn(s);
  }
  for (int lane = 1; lane < 8; ++lane) {
    if (!used[lane]) continue;
    if (!h->ev_join[lane]) YB_CHECK_CUDA(cudaEventCreateWithFlags(&h->ev_join[lane], cudaEventDisableTiming));
    YB_CHECK_CUDA(cudaEventRecord(h->ev_join[lane], h->lane_streams[lane]));
    YB_CHECK_CUDA(cudaStreamWaitEvent(stream, h->ev_join[lane], 0));
  }
}

static void run_ops_profiled(yb_handle* h, Executor* ex, cudaStream_t stream) {
  // eager, with an event pair around every op; conv share = sum over conv ops
  std::vector<cudaEvent_t> ev(ex->ops.size() + 1);
  for (auto& e : ev) YB_CHECK_CUDA(cudaEventCreate(&e));
  YB_CHECK_CUDA(cudaEventRecord(ev[0], stream));
  for (size_t i = 0; i < ex->ops.size(); ++i) {
    ex->ops[i].fn(stream);
    YB_CHECK_CUDA(cudaEventRecord(ev[i + 1], stream));
  }
  YB_CHECK_CUDA(cudaStreamSynchronize(stream));
  float total = 0.f, conv = 0.f;
  for (size_t i = 0; i < ex->ops.size(); ++i) {
    float ms = 0.f;
    YB_CHECK_CUDA(cudaEventElapsedTime(&ms, ev[i], ev[i + 1]));
    total += ms;
    ex->ops[i].last_ms = ms;
    if (ex->ops[i].is_conv) conv += ms;
  }
  h->last_total_ms = total;
  h->last_conv_ms = conv;
  for (auto& e : ev) cudaEventDestroy(e);
}

void yb_handle::forward(const float* d_x, int B, int H, int W, float* d_loc, float* d_conf, float* d_coef,
                        float* d_proto, cudaStream_t stream) {
  Executor* ex = get_executor(B, H, W);
  YB_CHECK_CUDA(cudaMemcpyAsync(ex->d_in, d_x, (size_t)B * 3 * H * W * 4, cudaMemcpyDeviceToDevice, stream));
  last_exec = ex;
  if (profiling) {
    run_ops_profiled(this, ex, stream);
  } else if (!use_graphs || ex->fwd_calls == 0) {
    run_ops(this, ex, stream);  // first call eager: validates launches, sets function attributes
  } else {
    if (!ex->graph_fwd) {
      cudaGraph_t g = nullptr;
      const int64_t before = lc.n;
      // capture on a private stream (the caller's stream may be the legacy default stream, which
      // cannot be captured); the instantiated graph is then launched into the caller's stream
      cudaStream_t cs = capture_stream();
      YB_CHECK_CUDA(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
      try {
        run_ops(this, ex, cs, true);
      } catch (...) {
        cudaStreamEndCapture(cs, &g);
        if (g) cudaGraphDestroy(g);
        throw;
      }
      YB_CHECK_CUDA(cudaStreamEndCapture(cs, &g));
      lc.n = before;  // capture does not launch
      YB_CHECK_CUDA(cudaGraphInstantiate(&ex->graph_fwd, g, 0));
      cudaGraphDestroy(g);
    }
    YB_CHECK_CUDA(cudaGraphLaunch(ex->graph_fwd, stream));
    lc.n += (int64_t)ex->ops.size();
  }
  ex->fwd_calls++;
  const void* src[4] = {ex->loc, ex->conf, ex->coef, ex->proto};
  void* dst[4] = {d_loc, d_conf, d_coef, d_proto};
  size_t bytes[4] = {(size_t)B * ex->P * 4 * 4, (size_t)B * ex->P * cfg.num_classes * 4,
                     (size_t)B * ex->P * cfg.mask_dim * 4, (size_t)B * ex->ph * ex->pw * cfg.mask_dim * 4};
  launch_multi_copy(src, dst, bytes, 4, stream, &lc);
}

void yb_handle::infer(const float* d_x, int B, int H, int W, int cross_class, int max_out, float* d_box,
                      float* d_coef_out, int64_t* d_cls, float* d_score, int32_t* d_count, float* d_proto,
                      cudaStream_t stream) {
  Executor* ex = get_executor(B, H, W);
  infer_on(ex, nullptr, d_x, cross_class, max_out, d_box, d_coef_out, d_cls, d_score, d_count, d_proto, stream);
}

void yb_handle::infer_frame_list(const uint8_t* const* frames, const int32_t* hw, int B, int H, int W, int mode,
                                 const float* mean_bgr, const float* std_bgr, int cross_class, int max_out,
                                 float* d_box, float* d_coef_out, int64_t* d_cls, float* d_score, int32_t* d_count,
                                 float* d_proto, cudaStream_t stream) {
  Executor* ex = get_executor(B, H, W);
  if (!ex->d_frame_table) ex->d_frame_table = (FrameRef*)dmalloc(ex->allocs, (size_t)B * sizeof(FrameRef));
  char key[256];
  snprintf(key, sizeof(key), "m%d %a %a %a / %a %a %a", mode, mean_bgr[0], mean_bgr[1], mean_bgr[2], std_bgr[0],
           std_bgr[1], std_bgr[2]);
  auto it = ex->frame_inputs.find(key);
  if (it == ex->frame_inputs.end()) {
    Executor::FrameInput fi;
    LaunchCounter* lc = &this->lc;
    const FrameRef* table = ex->d_frame_table;
    if (cfg.precision == YB_PREC_F32) {
      // no tensor-core stem to fuse into: FastBaseTransform into d_in, then the network's own stem
      float* d_in = ex->d_in;
      std::array<float, 3> mean{mean_bgr[0], mean_bgr[1], mean_bgr[2]}, stdv{std_bgr[0], std_bgr[1], std_bgr[2]};
      fi.entry.name = "fast_base_transform frame list";
      fi.entry.fn = [=](cudaStream_t s) {
        launch_fast_base_transform_list(table, B, H, W, mode, mean.data(), stdv.data(), d_in, s, lc);
      };
    } else {
      YB_REQUIRE(!ex->stem_plans.empty() && !ex->ops.empty(), "yb_infer_frame_list: the network has no tensor-core stem");
      StemTcPlan* sp = stem_tc_plan_create_frame_list(ex->stem_plans[0], table, mode, mean_bgr, std_bgr);
      ex->stem_plans.push_back(sp);
      fi.stem = sp;
      fi.entry.name = ex->ops[0].name + " frame list";
      fi.entry.fn = [sp, lc](cudaStream_t s) { launch_stem_tc(sp, s, lc); };
      fi.replaces_stem = true;
    }
    it = ex->frame_inputs.emplace(key, std::move(fi)).first;
  }
  // one entry per image, pointing at the caller's frame: nothing is copied but the table itself
  std::vector<FrameRef> table(B);
  for (int b = 0; b < B; ++b) table[b] = frame_ref(frames[b], hw[2 * b], hw[2 * b + 1], H, W);
  infer_on(ex, &it->second, table.data(), cross_class, max_out, d_box, d_coef_out, d_cls, d_score, d_count, d_proto,
           stream);
}

// Forward + Detect on an executor; fin == null takes NCHW fp32 input d_x into d_in, otherwise the host FrameRef table
// d_x into ex->d_frame_table.  Each input keeps its own captured graphs.
void yb_handle::infer_on(Executor* ex, Executor::FrameInput* fin, const void* d_x, int cross_class, int max_out,
                         float* d_box, float* d_coef_out, int64_t* d_cls, float* d_score, int32_t* d_count,
                         float* d_proto, cudaStream_t stream) {
  const int B = ex->B, H = ex->H, W = ex->W;
  DetectParams dp;
  dp.B = B;
  dp.P = ex->P;
  dp.num_classes = cfg.num_classes;
  dp.mask_dim = cfg.mask_dim;
  dp.top_k = cfg.nms_top_k;
  dp.conf_thresh = cfg.nms_conf_thresh;
  dp.nms_thresh = cfg.nms_thresh;
  dp.max_dets = cfg.max_num_detections;
  dp.conf_is_logits = 1;
  dp.cross_class = cross_class & 0xFF;
  dp.second_threshold = (cross_class & YB_NMS_FLAG_SECOND_THRESHOLD) ? 1 : 0;
  dp.max_size = (float)cfg.max_size;
  dp.max_out = max_out;
  // Detect buffers: allocated once per executor at the largest row count any NMS mode can ask for, so toggling
  // net.detect.use_cross_class_nms / use_fast_nms between calls neither re-allocates nor leaks
  const int cap = std::max(cfg.nms_top_k, cfg.max_num_detections);
  YB_REQUIRE(max_out >= 1 && max_out <= cap, "yb_infer: max_out must be in [1, max(nms_top_k, max_num_detections)]");
  if (!ex->det_ws) {
    ex->det_ws = dmalloc(ex->allocs, detect_workspace_bytes(B, ex->P, cfg.num_classes, cfg.nms_top_k));
    detect_workspace_bind(&ex->dws, ex->det_ws, B, ex->P, cfg.num_classes, cfg.nms_top_k);
    ex->det_box = (float*)dmalloc(ex->allocs, (size_t)B * cap * 4 * 4);
    ex->det_coef = (float*)dmalloc(ex->allocs, (size_t)B * cap * cfg.mask_dim * 4);
    ex->det_cls = (int64_t*)dmalloc(ex->allocs, (size_t)B * cap * 8);
    ex->det_score = (float*)dmalloc(ex->allocs, (size_t)B * cap * 4);
    ex->det_count = (int32_t*)dmalloc(ex->allocs, (size_t)B * 4);
    ex->det_cap = cap;
  }
  Executor::InferGraph& ig = (fin ? fin->graphs : ex->infer_graphs)[(cross_class & 0xFFF) | (max_out << 12)];
  auto run_all = [&](cudaStream_t s, bool branches) {
    run_ops(this, ex, s, branches, fin);
    launch_detect(dp, ex->loc, ex->conf, ex->coef, ex->priors, ex->dws, ex->det_box, ex->det_coef, ex->det_cls,
                  ex->det_score, ex->det_count, s, &lc);
  };
  if (fin)
    // pageable source: staged before the call returns, so the host table may go away at once.  Stream-ordered after
    // the previous call (CallGuard), so an earlier replay has read the table before it is overwritten.
    YB_CHECK_CUDA(cudaMemcpyAsync(ex->d_frame_table, d_x, (size_t)B * sizeof(FrameRef), cudaMemcpyHostToDevice, stream));
  else
    YB_CHECK_CUDA(cudaMemcpyAsync(ex->d_in, d_x, (size_t)B * 3 * H * W * 4, cudaMemcpyDeviceToDevice, stream));
  last_exec = ex;
  if (!use_graphs || ig.calls == 0) {
    run_all(stream, false);   // first call of this mode eager: validates launches, sets function attributes
  } else {
    if (!ig.exec) {
      cudaGraph_t g = nullptr;
      const int64_t before = lc.n;
      cudaStream_t cs = capture_stream();
      YB_CHECK_CUDA(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
      try {
        run_all(cs, true);
      } catch (...) {
        cudaStreamEndCapture(cs, &g);
        if (g) cudaGraphDestroy(g);
        throw;
      }
      YB_CHECK_CUDA(cudaStreamEndCapture(cs, &g));
      lc.n = before;
      YB_CHECK_CUDA(cudaGraphInstantiate(&ig.exec, g, 0));
      cudaGraphDestroy(g);
    }
    YB_CHECK_CUDA(cudaGraphLaunch(ig.exec, stream));
    const int64_t net_ops = (int64_t)ex->ops.size() + ((fin && !fin->replaces_stem) ? 1 : 0);
    lc.n += net_ops + (dp.cross_class == YB_NMS_CROSS_CLASS ? 2 : 3);
  }
  ig.calls++;
  const void* src[6] = {ex->det_box, ex->det_coef, ex->det_cls, ex->det_score, ex->det_count, ex->proto};
  void* dst[6] = {d_box, d_coef_out, d_cls, d_score, d_count, d_proto};
  size_t bytes[6] = {(size_t)B * max_out * 16, (size_t)B * max_out * cfg.mask_dim * 4, (size_t)B * max_out * 8,
                     (size_t)B * max_out * 4, (size_t)B * 4, (size_t)B * ex->ph * ex->pw * cfg.mask_dim * 4};
  launch_multi_copy(src, dst, bytes, 6, stream, &lc);
}
