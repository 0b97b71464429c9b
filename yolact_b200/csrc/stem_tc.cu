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
};

// SPLIT (YB_PREC_F16X3): the patch is written as a hi and a lo fp16 tile, the weights come as [Cout][hi(Kpad) | lo(Kpad)],
// three MMA passes (hi*hi into one accumulator, lo*hi + hi*lo into a second one) and the output pixel is [hi(COUT) | lo(COUT)].
template <int KS, int STRIDE, int PAD, int COUT, int WG, bool SPLIT>
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
  {
    const int row = tid & 127;
    const int wg = tid >> 7;   // worker group: which k-groups of the patch this thread gathers
    const long long m = (long long)blockIdx.x * ST_M + row;
    const bool valid = m < p.M;
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
      const long long m = (long long)blockIdx.x * ST_M + row;
      if (m >= p.M) continue;
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

template <int KS, int STRIDE, int PAD, int COUT, int WG, bool SPLIT>
void launch_variant(const StemParams& prm, cudaStream_t stream) {
  constexpr int K = 3 * KS * KS;
  constexpr int ATOMS = (K + 63) / 64;
  const size_t smem = (size_t)(SPLIT ? 2 : 1) * ATOMS * (ST_M * 128 + COUT * 128) + 1024;
  static PerDeviceOnce attr;
  if (attr.first())
    YB_CHECK_CUDA(cudaFuncSetAttribute(stem_tc_kernel<KS, STRIDE, PAD, COUT, WG, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem));
  const unsigned grid = (unsigned)((prm.M + ST_M - 1) / ST_M);
  stem_tc_kernel<KS, STRIDE, PAD, COUT, WG, SPLIT><<<grid, 128 * WG, smem, stream>>>(prm);
}

}  // namespace

struct StemTcPlan {
  StemParams prm;
  int ks, stride, pad, cout;
  int split = 0;
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

void stem_tc_plan_destroy(StemTcPlan* plan) { delete plan; }

void launch_stem_tc(const StemTcPlan* plan, cudaStream_t stream, LaunchCounter* lc) {
  if (plan->split) {
    // the split stem holds 144 KB of operand tiles (one CTA per SM): two worker threads per pixel double the warps
    // that hide the gather's latency
    if (plan->ks == 7)
      launch_variant<7, 2, 3, 64, 2, true>(plan->prm, stream);
    else
      launch_variant<3, 1, 1, 32, 1, true>(plan->prm, stream);
  } else if (plan->ks == 7) {
    launch_variant<7, 2, 3, 64, 1, false>(plan->prm, stream);
  } else {
    launch_variant<3, 1, 1, 32, 1, false>(plan->prm, stream);
  }
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

}  // namespace yb
