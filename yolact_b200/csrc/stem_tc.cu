// Network stem on the tensor cores (wgmma): conv KxK over the 3-channel NCHW fp32 input frame (+ folded BN +
// activation) -> NHWC fp16.  ResNet: 7x7/2 pad 3, 3->64, ReLU (backbone.py:77-79,129-131).  Darknet: 3x3/1 pad 1,
// 3->32, LeakyReLU(0.1) (backbone.py:267, :222-233).
//
// Cin = 3 is useless for TMA (6 bytes per pixel) so the A operand is built by the CUDA cores:
// each of the 128 worker threads owns one output pixel, gathers its KxKx3 patch straight from the
// fp32 NCHW frame (zero padding by predication, layout conversion and fp32->fp16 cast fused in),
// (with WG = 2 worker warpgroups, as in the split-precision 7x7 stem, two threads share a pixel: alternate 16-byte
// k-groups of the patch -- more warps in flight for the latency-bound gather)
// and writes it as one K-major SWIZZLE_128B row of the wgmma A tile in shared memory
// (k = c*K*K + r*K + s, the OIHW flattening, so the weights need no permutation).  Thread 0 TMA-loads the
// [Cout][Kpad] weight tile meanwhile; then warpgroup w runs ceil(K/16) wgmmas (M = 64, N = Cout) for the 64-row
// halves w, w + WG of the tile and stores its rows' pixels from the accumulator registers.
// Several CTAs per SM overlap gather / MMA / epilogue of different tiles.
//
// Frame-list source (FRAME_LIST, yb_infer_frame_list and yb_infer_frames): the input is a list of [fh][fw][3] uint8 BGR
// frames, each of its own size, and FastBaseTransform (resize to H x W, transform, BGR -> RGB) happens in the loader, so
// no NCHW fp32 input is ever written.  The 128 rows of a tile are then an 8 x 16 block of output pixels of one image.
// A CTA reads its image's FrameRef (frame, fh, fw, scales) from a device table; nothing else about the launch depends on
// the frame sizes, so one plan and one graph serve any mix of them.  The tile's receptive field is a rectangle of the
// resized image (FrameWindow: 21 x 37 pixels for 7x7/2, 10 x 18 for 3x3/1): all threads first fill a [3][ROWS][COLS]
// fp32 window of it in shared memory with common.cuh xform_pixel (zero outside the image: the conv's padding), then the
// gather above reads the window instead of global memory.  A window pixel is shared by up to 16 patches, so staging
// computes each resized pixel about 1.5 times per CTA where a direct gather would compute it once per tap.
// Each output pixel's patch, and so its wgmma row and its output, is bit-identical to the NCHW path's on
// fast_base_transform's output.
#include "tc_common.cuh"

namespace yb {

using namespace tc;

namespace {

constexpr int ST_M = 128;
// threads = 128 * WG workers (warpgroups)

struct alignas(64) StemParams {
  CUtensorMap tmW;
  const float* x;
  const float* bias;
  __half* y;
  int B, H, W, Ho, Wo;
  int cpad;               // channels per output pixel (>= COUT, multiple of 8; channels COUT..cpad-1 are written as zeros so
                          // that a tensor-core conv with Cin % 64 == 0 can consume a 32-channel stem, e.g. Darknet's)
  long long M;
  int act;
  float out_scale;   // split: weights are pre-multiplied by 1 / out_scale (a power of two)
  // frame-list source: image b is frame_list[b], resized to H x W
  int xform_mode;
  XformAffine aff;
  int tiles_x, tiles_y;   // output tiles of FT_H x FT_W pixels per image
  const FrameRef* frame_list;   // [B] entries
};

constexpr int FT_H = 8, FT_W = 16;   // frame list: a tile's 128 rows are FT_H x FT_W output pixels (row = y * FT_W + x)
template <int KS, int STRIDE>
struct FrameWindow {   // resized pixels a tile reads: [3][ROWS][COLS] fp32
  static constexpr int ROWS = (FT_H - 1) * STRIDE + KS, COLS = (FT_W - 1) * STRIDE + KS;
  static constexpr int BYTES = 3 * ROWS * COLS * 4;
};

// SPLIT (YB_PREC_F16X3): the patch is written as a hi and a lo fp16 tile, the weights come as [Cout][hi(Kpad) | lo(Kpad)],
// three MMA passes (hi*hi into one accumulator, lo*hi + hi*lo into a second one) and the output pixel is [hi(COUT) | lo(COUT)].
template <int KS, int STRIDE, int PAD, int COUT, int WG, bool SPLIT, bool FRAME_LIST>
__global__ void __launch_bounds__(128 * WG)
stem_tc_kernel(const __grid_constant__ StemParams p) {
  constexpr int NPL = SPLIT ? 2 : 1;
  constexpr int K = 3 * KS * KS;
  constexpr int ATOMS = (K + 63) / 64;
  constexpr int KSTEPS = (K + 15) / 16;
  constexpr int A_ATOM_BYTES = ST_M * 128;
  constexpr int B_ATOM_BYTES = COUT * 128;

  extern __shared__ uint8_t smem_dyn[];
  __shared__ uint64_t b_full;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
  uint8_t* sA = smem;                               // [plane][atom]
  uint8_t* sB = smem + NPL * ATOMS * A_ATOM_BYTES;  // [plane][atom]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    mbar_init(&b_full, 1);
    fence_barrier_init();
    mbar_expect_tx(&b_full, NPL * ATOMS * B_ATOM_BYTES);
    for (int pl = 0; pl < NPL; ++pl)
      for (int a = 0; a < ATOMS; ++a)
        tma_load_3d(sB + (pl * ATOMS + a) * B_ATOM_BYTES, &p.tmW, &b_full, pl * ATOMS * 64 + a * 64, 0, 0);
  }
  using Win = FrameWindow<KS, STRIDE>;
  int fb = 0, fty = 0, ftx = 0;   // frame list: this tile's image and tile coordinates
  if constexpr (FRAME_LIST) {
    int t = blockIdx.x;
    ftx = t % p.tiles_x;
    t /= p.tiles_x;
    fty = t % p.tiles_y;
    fb = t / p.tiles_y;
    float* win = reinterpret_cast<float*>(sB + NPL * ATOMS * B_ATOM_BYTES);
    const int y0 = fty * FT_H * STRIDE - PAD, x0 = ftx * FT_W * STRIDE - PAD;
    const FrameRef f = p.frame_list[fb];   // this image's frame, size and resize scales
    for (int i = tid; i < Win::ROWS * Win::COLS; i += 128 * WG) {
      const int y = y0 + i / Win::COLS, x = x0 + i % Win::COLS;
      float rgb[3] = {0.f, 0.f, 0.f};
      if (y >= 0 && y < p.H && x >= 0 && x < p.W)
        xform_pixel(f.frame, f.fw, xform_tap(y, p.H, f.fh, f.scale_h), xform_tap(x, p.W, f.fw, f.scale_w), p.xform_mode,
                    p.aff, rgb);
#pragma unroll
      for (int c = 0; c < 3; ++c) win[c * Win::ROWS * Win::COLS + i] = rgb[c];
    }
    __syncthreads();
  }
  {
    const int row = tid & 127;
    const int wg = tid >> 7;   // worker group: which k-groups of the patch this thread gathers
    long long m;
    bool valid;
    if constexpr (FRAME_LIST) {
      const int ho = fty * FT_H + row / FT_W, wo = ftx * FT_W + row % FT_W;
      valid = ho < p.Ho && wo < p.Wo;
      m = ((long long)fb * p.Ho + ho) * p.Wo + wo;
      // tap (0, 0) of this pixel in the window, which holds the zero padding: no predication
      const float* xw = reinterpret_cast<const float*>(sB + NPL * ATOMS * B_ATOM_BYTES) +
                        (row / FT_W) * STRIDE * Win::COLS + (row % FT_W) * STRIDE;
      // the NCHW gather below with the window as its source (kept as two loops: through one shared loop the NCHW
      // instances compile to different SASS)
#pragma unroll
      for (int kg = 0; kg < ATOMS * 8; ++kg) {
        if (WG > 1 && (kg % WG) != wg) continue;   // warp-uniform
        uint4 pk, pkl;
        __half2* h2 = reinterpret_cast<__half2*>(&pk);
        __half2* l2 = reinterpret_cast<__half2*>(&pkl);
#pragma unroll
        for (int j2 = 0; j2 < 4; ++j2) {
          float v[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int k = kg * 8 + j2 * 2 + e;   // compile-time after unrolling
            float val = 0.f;
            if (k < K) {
              const int c = k / (KS * KS), r = (k % (KS * KS)) / KS, s = k % KS;
              val = xw[(c * Win::ROWS + r) * Win::COLS + s];
            }
            v[e] = val;
          }
          if (SPLIT) split2_from_f32(v[0], v[1], h2[j2], l2[j2]);
          else h2[j2] = __halves2half2(from_f32<__half>(v[0]), from_f32<__half>(v[1]));
        }
        const int atom = kg >> 3;
        const uint32_t aoff = sw128_off(row, kg & 7);
        *reinterpret_cast<uint4*>(sA + atom * A_ATOM_BYTES + aoff) = pk;
        if (SPLIT) *reinterpret_cast<uint4*>(sA + (ATOMS + atom) * A_ATOM_BYTES + aoff) = pkl;
      }
    } else {
      m = (long long)blockIdx.x * ST_M + row;
      valid = m < p.M;
      int b = 0, ho = 0, wo = 0;
      if (valid) {
        wo = (int)(m % p.Wo);
        const long long t = m / p.Wo;
        ho = (int)(t % p.Ho);
        b = (int)(t / p.Ho);
      }
      const int hb = ho * STRIDE - PAD, wb = wo * STRIDE - PAD;
      unsigned rmask = 0, cmask = 0;
#pragma unroll
      for (int r = 0; r < KS; ++r) {
        if (valid && hb + r >= 0 && hb + r < p.H) rmask |= 1u << r;
        if (valid && wb + r >= 0 && wb + r < p.W) cmask |= 1u << r;
      }
      const size_t plane = (size_t)p.H * p.W;
      const float* xb = p.x + (size_t)b * 3 * plane + (long long)hb * p.W + wb;  // may point before the frame: guarded
      // the frame-list branch above repeats this loop with the window as its source: the two must keep the same k order
      // and encoding, or yb_infer_frame_list stops being bit-identical to yb_infer on fast_base_transform's output
#pragma unroll
      for (int kg = 0; kg < ATOMS * 8; ++kg) {
        if (WG > 1 && (kg % WG) != wg) continue;   // warp-uniform
        uint4 pk, pkl;
        __half2* h2 = reinterpret_cast<__half2*>(&pk);
        __half2* l2 = reinterpret_cast<__half2*>(&pkl);
#pragma unroll
        for (int j2 = 0; j2 < 4; ++j2) {
          float v[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int k = kg * 8 + j2 * 2 + e;   // compile-time after unrolling
            float val = 0.f;
            if (k < K) {
              const int c = k / (KS * KS), r = (k % (KS * KS)) / KS, s = k % KS;
              if (((rmask >> r) & 1u) && ((cmask >> s) & 1u)) val = __ldg(xb + (size_t)c * plane + r * p.W + s);
            }
            v[e] = val;
          }
          if (SPLIT) split2_from_f32(v[0], v[1], h2[j2], l2[j2]);
          else h2[j2] = __halves2half2(from_f32<__half>(v[0]), from_f32<__half>(v[1]));
        }
        const int atom = kg >> 3;
        const uint32_t aoff = sw128_off(row, kg & 7);
        *reinterpret_cast<uint4*>(sA + atom * A_ATOM_BYTES + aoff) = pk;
        if (SPLIT) *reinterpret_cast<uint4*>(sA + (ATOMS + atom) * A_ATOM_BYTES + aoff) = pkl;
      }
    }
    __half* yrow = p.y + m * (long long)(p.cpad * NPL);
    if (valid && wg == 0)
      for (int c0 = COUT; c0 < p.cpad; c0 += 8) {   // zero padding channels (both planes)
        *reinterpret_cast<uint4*>(yrow + c0) = make_uint4(0u, 0u, 0u, 0u);
        if (SPLIT) *reinterpret_cast<uint4*>(yrow + p.cpad + c0) = make_uint4(0u, 0u, 0u, 0u);
      }
  }
  fence_proxy_async();   // generic-proxy smem writes -> visible to wgmma (async proxy)
  __syncthreads();
  mbar_wait(&b_full, 0);

  // ---- MMA + epilogue: 64-row half h of the tile -> bias -> activation -> this thread's channel pairs of its two rows
  const int wgi = warp >> 2, wq = warp & 3;
  for (int h = wgi; h < 2; h += WG) {
    float acc[NPL][COUT / 2];
#pragma unroll
    for (int pl = 0; pl < NPL; ++pl)
#pragma unroll
      for (int i = 0; i < COUT / 2; ++i) acc[pl][i] = 0.f;
    wgmma_fence();
    mma_passes<COUT, KSTEPS, SPLIT>(
        acc[0], acc[NPL - 1],
        [&](int pl, int j) {
          return make_sw128_desc(smem_u32(sA + (pl * ATOMS + (j >> 2)) * A_ATOM_BYTES + h * 64 * 128)) + (uint64_t)(2 * (j & 3));
        },
        [&](int pl, int j) {
          return make_sw128_desc(smem_u32(sB + (pl * ATOMS + (j >> 2)) * B_ATOM_BYTES)) + (uint64_t)(2 * (j & 3));
        });
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int pl = 0; pl < NPL; ++pl) fence_regs<COUT / 2>(acc[pl]);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = h * 64 + wq * 16 + (lane >> 2) + 8 * hh;
      long long m;
      if constexpr (FRAME_LIST) {
        const int ho = fty * FT_H + row / FT_W, wo = ftx * FT_W + row % FT_W;
        if (ho >= p.Ho || wo >= p.Wo) continue;
        m = ((long long)fb * p.Ho + ho) * p.Wo + wo;
      } else {
        m = (long long)blockIdx.x * ST_M + row;
        if (m >= p.M) continue;
      }
      __half* yrow = p.y + m * (long long)(p.cpad * NPL);
#pragma unroll
      for (int j = 0; j < COUT / 8; ++j) {
        const int col = 8 * j + 2 * (lane & 3);
        const int i = 4 * j + 2 * hh;
        const float a0 = SPLIT ? split_combine(acc[0][i], acc[NPL - 1][i]) : acc[0][i];
        const float a1 = SPLIT ? split_combine(acc[0][i + 1], acc[NPL - 1][i + 1]) : acc[0][i + 1];
        const float v0 = apply_act(scale_bias<SPLIT>(a0, p.out_scale, p.bias ? __ldg(p.bias + col) : 0.f), p.act);
        const float v1 = apply_act(scale_bias<SPLIT>(a1, p.out_scale, p.bias ? __ldg(p.bias + col + 1) : 0.f), p.act);
        __half2 hi, lo;
        if (SPLIT) split2_from_f32(v0, v1, hi, lo);
        else hi = __halves2half2(from_f32<__half>(v0), from_f32<__half>(v1));
        *reinterpret_cast<__half2*>(yrow + col) = hi;
        if (SPLIT) *reinterpret_cast<__half2*>(yrow + p.cpad + col) = lo;
      }
    }
  }
}

template <int KS, int STRIDE, int PAD, int COUT, int WG, bool SPLIT, bool FRAME_LIST>
void launch_variant(const StemParams& prm, cudaStream_t stream) {
  constexpr int K = 3 * KS * KS;
  constexpr int ATOMS = (K + 63) / 64;
  const size_t smem = (size_t)(SPLIT ? 2 : 1) * ATOMS * (ST_M * 128 + COUT * 128) + 1024 +
                      (FRAME_LIST ? FrameWindow<KS, STRIDE>::BYTES : 0);
  static PerDeviceOnce attr;
  if (attr.first())
    YB_CHECK_CUDA(cudaFuncSetAttribute(stem_tc_kernel<KS, STRIDE, PAD, COUT, WG, SPLIT, FRAME_LIST>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const unsigned grid = FRAME_LIST ? (unsigned)(prm.B * prm.tiles_y * prm.tiles_x) : (unsigned)((prm.M + ST_M - 1) / ST_M);
  stem_tc_kernel<KS, STRIDE, PAD, COUT, WG, SPLIT, FRAME_LIST><<<grid, 128 * WG, smem, stream>>>(prm);
}

template <bool FRAME_LIST>
void launch_stem(const StemParams& prm, int ks, bool split, cudaStream_t stream) {
  if (split) {
    // the split stem holds 144 KB of operand tiles (one CTA per SM): two worker threads per pixel double the warps
    // that hide the gather's latency
    if (ks == 7)
      launch_variant<7, 2, 3, 64, 2, true, FRAME_LIST>(prm, stream);
    else
      launch_variant<3, 1, 1, 32, 1, true, FRAME_LIST>(prm, stream);
  } else if (ks == 7) {
    launch_variant<7, 2, 3, 64, 1, false, FRAME_LIST>(prm, stream);
  } else {
    launch_variant<3, 1, 1, 32, 1, false, FRAME_LIST>(prm, stream);
  }
}

}  // namespace

struct StemTcPlan {
  StemParams prm;
  int ks, stride, pad, cout;
  int split = 0;
  bool frame_list = false;
};

bool stem_tc_supported(int ks, int stride, int pad, int cin, int cout) {
  return cin == 3 && ((ks == 7 && stride == 2 && pad == 3 && cout == 64) || (ks == 3 && stride == 1 && pad == 1 && cout == 32));
}

int stem_tc_kpad(int ks) { return ((3 * ks * ks + 63) / 64) * 64; }

StemTcPlan* stem_tc_plan_create(const float* x_nchw, const __half* w_packed, const float* bias, __half* y, int B, int H,
                                int W, int ks, int stride, int pad, int cout, int act, int split, float out_scale, int cpad) {
  YB_REQUIRE(stem_tc_supported(ks, stride, pad, 3, cout), "stem_tc: unsupported stem shape");
  auto* plan = new StemTcPlan();
  StemParams& q = plan->prm;
  memset(&q, 0, sizeof(q));
  plan->ks = ks;
  plan->stride = stride;
  plan->pad = pad;
  plan->cout = cout;
  q.x = x_nchw;
  q.bias = bias;
  q.y = y;
  q.B = B;
  q.H = H;
  q.W = W;
  q.Ho = (H + 2 * pad - ks) / stride + 1;
  q.Wo = (W + 2 * pad - ks) / stride + 1;
  q.M = (long long)B * q.Ho * q.Wo;
  q.cpad = cpad > cout ? cpad : cout;
  YB_REQUIRE(q.cpad % 8 == 0, "stem_tc: the padded channel count must be a multiple of 8");
  q.act = act;
  q.out_scale = split ? out_scale : 1.f;
  plan->split = split ? 1 : 0;
  const int kpad = stem_tc_kpad(ks);
  const uint64_t kp = (uint64_t)kpad * (split ? 2 : 1);   // [cout][hi(kpad) | lo(kpad)]
  uint64_t dims[3] = {kp, (uint64_t)cout, 1};
  uint64_t str[2] = {kp * 2, kp * cout * 2};
  uint32_t box[3] = {64, (uint32_t)cout, 1};
  encode_map_f16(&q.tmW, w_packed, 3, dims, str, box);
  return plan;
}

StemTcPlan* stem_tc_plan_create_frame_list(const StemTcPlan* net_stem, const FrameRef* d_table, int mode,
                                           const float* mean_bgr, const float* std_bgr) {
  YB_REQUIRE(d_table, "stem_tc: no frame table");
  YB_REQUIRE(!net_stem->frame_list, "stem_tc: the frame stem is derived from the network's NCHW stem");
  YB_REQUIRE(mode >= YB_XFORM_NORMALIZE && mode <= YB_XFORM_NONE, "stem_tc: unknown transform mode");
  const int tiles_x = ceil_div(net_stem->prm.Wo, FT_W), tiles_y = ceil_div(net_stem->prm.Ho, FT_H);
  YB_REQUIRE((long long)net_stem->prm.B * tiles_y * tiles_x < (1ll << 31), "stem_tc: frame batch too large for one grid");
  auto* plan = new StemTcPlan(*net_stem);
  StemParams& q = plan->prm;
  plan->frame_list = true;
  q.x = nullptr;
  q.xform_mode = mode;
  for (int c = 0; c < 3; ++c) {
    q.aff.mean[c] = mean_bgr[c];
    q.aff.stdv[c] = std_bgr[c];
  }
  q.tiles_x = tiles_x;
  q.tiles_y = tiles_y;
  q.frame_list = d_table;
  return plan;
}

void stem_tc_plan_destroy(StemTcPlan* plan) { delete plan; }

void launch_stem_tc(const StemTcPlan* plan, cudaStream_t stream, LaunchCounter* lc) {
  if (plan->frame_list)
    launch_stem<true>(plan->prm, plan->ks, plan->split, stream);
  else
    launch_stem<false>(plan->prm, plan->ks, plan->split, stream);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

}  // namespace yb
