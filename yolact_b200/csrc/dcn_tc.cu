// Fused DCNv2 (modulated deformable convolution, any kh x kw kernel and geometry, deformable groups of a multiple of 64
// channels) on the tensor cores (wgmma): deformable gather ->
// shared-memory A stage -> tensor-core contraction -> bias + ReLU, ONE kernel, no column buffer.
//
// Reference: DCN.forward (external/DCNv2/dcn_v2.py:118-128), modulated_deformable_im2col_gpu_kernel
// (external/DCNv2/src/cuda/dcn_v2_im2col_cuda.cu:125-195, bilinear sampler :25-54) followed by the batched SGEMM + bias
// of dcn_v2_cuda_forward (src/cuda/dcn_v2_cuda.cu:123-163).  The reference materialises the sampled columns
// [B, taps*C, Ho*Wo] fp32 in HBM between the two.  Here they never leave the SM:
//
//   GEMM view   D[128 output pixels, BN couts] = sum over taps t (kh*kw) and 64-channel chunks kc of
//               A_t,kc[128, 64] * W[BN, t*C + kc*64 .. +64]^T,
//               A_t,kc[m, c] = mask(m,t,g) * bilinear(x, pos(m,t,g))[kc*64 + c]      (fp32 math, reference op order)
//               with g = kc*64 / (C/dg) the deformable group of the chunk: (C/dg) % 64 == 0, so a chunk never
//               straddles two groups
//   warp 8      TMA producer of the weight tiles (B operand, [Cout][taps*C] K-major)
//   warps 0..7  two warpgroups; each gathers the A rows of its 64-row half of the tile and multiplies them with wgmma
//               while it gathers the next k-block.  Gather: warp w owns 16 tile rows.  Once per (tap, group), lanes 0..15 each compute the sampling geometry
//               of ONE row (4 corner offsets, 4 bilinear weights, the modulation mask) from its offset/mask channels; for
//               every 64-channel chunk the geometry reaches the lanes that need it by WARP SHUFFLE (8 lanes share a
//               row: one 16-byte vector of 8 channels each), the four corners are fetched with 16-byte loads, blended
//               (fp32 in the split mode, packed half2 in the fp16 mode) and written as one swizzled 16-byte piece of the K-major SWIZZLE_128B A tile -- the layout
//               wgmma consumes directly.  Geometry is computed once per (pixel, tap, group), not once
//               per (pixel, tap, 8 channels).
//   epilogue    each warpgroup: accumulator registers -> (* out_scale) + bias -> ReLU -> its rows' channel pairs.
//   SPLIT       (YB_PREC_F16X3) x and y are [hi(C) | lo(C)] pairs, the sample is hi + lo, the A stage holds a hi (fp16)
//               and a lo (2^11-scaled fp16) tile, the weights [Cout][hi(taps*C) | lo(taps*C)], three MMA passes per
//               k-block.
#include "tc_common.cuh"

namespace yb {

using namespace tc;

namespace {

constexpr int DM = 128;                 // tile rows (output pixels)
constexpr int DK = 64;                  // channels per k-block (one 128-byte swizzle row)
constexpr int A_TILE = DM * DK * 2;     // 16 KB
constexpr int GATHER_WARPS = 8;
constexpr int DTHREADS = 32 * GATHER_WARPS + 32;
constexpr int MAX_DSTAGES = 6;

struct alignas(64) DcnParams {
  CUtensorMap tmW;
  const __half* x;
  const float* om;      // [M, 3*dg*taps]: per group 2*taps offsets (dh, dw interleaved per tap), then per group taps
                        // mask logits / masks
  const float* bias;
  __half* y;
  int B, H, W, C, Ho, Wo, Cout;
  long long M;
  yb_dcn_params g;
  int taps;
  int act, mask_logits;
  int stages, kchunks;
  int gchunks;          // k-blocks per deformable group: (C / dg) / 64
  float out_scale;
};

template <int BN, bool SPLIT>
__global__ void __launch_bounds__(DTHREADS)
dcn_tc_kernel(const __grid_constant__ DcnParams p) {
  constexpr int NPL = SPLIT ? 2 : 1;
  constexpr int B_PLANE = BN * DK * 2;
  constexpr int STAGE = NPL * (A_TILE + B_PLANE);
  static_assert(NPL * BN / 2 <= 128, "accumulator tile exceeds the register budget");

  extern __shared__ uint8_t smem_dyn[];
  __shared__ uint64_t b_full[MAX_DSTAGES], empty_bar[MAX_DSTAGES];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int stages = p.stages;
  const int num_kb = p.taps * p.kchunks;
  const long long m0 = (long long)blockIdx.x * DM;
  const int n0 = blockIdx.y * BN;

  if (tid == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(&b_full[s], 1);
      mbar_init(&empty_bar[s], 2);   // both warpgroups have read the weight tile
    }
    fence_barrier_init();
    tma_prefetch_desc(&p.tmW);
  }
  __syncthreads();

  if (warp == GATHER_WARPS) {
    // ===================== weight tiles (TMA) =====================
    if (lane == 0) {
      for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % stages, it = kb / stages;
        mbar_wait(&empty_bar[s], (uint32_t)(it & 1) ^ 1u);
        const int tap = kb / p.kchunks, kc = kb - tap * p.kchunks;
        uint8_t* sb = smem + (size_t)s * STAGE + NPL * A_TILE;
        mbar_expect_tx(&b_full[s], (uint32_t)(NPL * B_PLANE));
#pragma unroll
        for (int pl = 0; pl < NPL; ++pl)
          tma_load_3d(sb + pl * B_PLANE, &p.tmW, &b_full[s], tap * p.C + kc * DK + pl * p.taps * p.C, n0, 0);
      }
    }
  } else {
    // ===================== gather warps =====================
    const int gw = warp;                            // 0..7: rows [16*gw, 16*gw + 16)
    const int wgi = warp >> 2;                      // warpgroup: rows [64*wgi, 64*wgi + 64)
    float acc[NPL][BN / 2];
#pragma unroll
    for (int pl = 0; pl < NPL; ++pl)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[pl][i] = 0.f;
    const int PS = NPL * p.C;                       // halfs per input pixel
    // geometry owner: lanes 0..15 <-> row 16*gw + lane
    const long long gm = m0 + gw * 16 + (lane & 15);
    const bool gvalid = (lane < 16) && (gm < p.M);
    int gb = 0, gho = 0, gwo = 0;
    if (gvalid) {
      gwo = (int)(gm % p.Wo);
      const long long t = gm / p.Wo;
      gho = (int)(t % p.Ho);
      gb = (int)(t / p.Ho);
    }
    const int dg = p.g.deformable_group;
    const float* gom = p.om + gm * (3 * dg * p.taps);
    const int img_base = gb * p.H * p.W;
    // this lane's items: 4 per k-block; item i -> row 16*gw + 4*i + (lane >> 3), 16-byte piece (lane & 7)
    const int piece = lane & 7;
    const int src_sub = lane >> 3;                  // + 4*i = geometry owner lane

    // Corner offsets are ALWAYS valid addresses (an out-of-range corner points at this image's pixel 0 and carries
    // weight 0, which is what the reference's `if (h_low >= 0 && ...) v = ...` amounts to): the corner loads of a
    // k-block are then unconditional and the compiler issues them back to back -- with a branch per corner every load
    // would wait for the previous one.
    // The modulation mask is folded into the four bilinear weights (one rounding of difference to the reference's
    // (sum) * mask, far below the fp16 / split resolution).
    int ao[4][4];        // [item][corner] pixel offsets of this lane's 4 rows, refreshed once per tap by shuffle
    float aw[4][4];      // [item][corner] weight * mask (split mode)
    __half2 hw[4][4];    // the same as broadcast half2 pairs (fp16 mode)
    int cur_key = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      const int s = kb % stages, it = kb / stages;
      const int tap = kb / p.kchunks, kc = kb - tap * p.kchunks;
      const int gr = kc / p.gchunks;
      if (tap * dg + gr != cur_key) {
        cur_key = tap * dg + gr;
        int o00 = img_base, o01 = img_base, o10 = img_base, o11 = img_base;
        float w00 = 0.f, w01 = 0.f, w10 = 0.f, w11 = 0.f;
        if (gvalid) {
          // dcn_v2_im2col_cuda.cu:151-189: h_im = h_in + i*dil + offset_h, w_im likewise; inside test (-1, H) x (-1, W)
          const int i = tap / p.g.kernel_w, j = tap - i * p.g.kernel_w;
          const float* goff = gom + gr * 2 * p.taps + 2 * tap;
          const float hh = __fadd_rn((float)(gho * p.g.stride_h - p.g.pad_h + i * p.g.dilation_h), __ldg(goff));
          const float ww = __fadd_rn((float)(gwo * p.g.stride_w - p.g.pad_w + j * p.g.dilation_w), __ldg(goff + 1));
          const float mv = __ldg(gom + 2 * dg * p.taps + gr * p.taps + tap);
          const float msk = p.mask_logits ? __fdiv_rn(1.f, __fadd_rn(1.f, expf(-mv))) : mv;
          if (hh > -1.f && ww > -1.f && hh < (float)p.H && ww < (float)p.W) {
            const int hl = (int)floorf(hh), wl = (int)floorf(ww);
            const int hhi = hl + 1, whi = wl + 1;
            const float lh = __fsub_rn(hh, (float)hl), lw = __fsub_rn(ww, (float)wl);
            const float uh = __fsub_rn(1.f, lh), uw = __fsub_rn(1.f, lw);
            if (hl >= 0 && wl >= 0) {
              o00 = img_base + hl * p.W + wl;
              w00 = __fmul_rn(__fmul_rn(uh, uw), msk);
            }
            if (hl >= 0 && whi <= p.W - 1) {
              o01 = img_base + hl * p.W + whi;
              w01 = __fmul_rn(__fmul_rn(uh, lw), msk);
            }
            if (hhi <= p.H - 1 && wl >= 0) {
              o10 = img_base + hhi * p.W + wl;
              w10 = __fmul_rn(__fmul_rn(lh, uw), msk);
            }
            if (hhi <= p.H - 1 && whi <= p.W - 1) {
              o11 = img_base + hhi * p.W + whi;
              w11 = __fmul_rn(__fmul_rn(lh, lw), msk);
            }
          }
        }
        // geometry owner lane -> the 8 lanes that gather that row (item i: row 16*gw + 4*i + (lane >> 3))
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int src = 4 * i + src_sub;
          ao[i][0] = __shfl_sync(0xffffffffu, o00, src);
          ao[i][1] = __shfl_sync(0xffffffffu, o01, src);
          ao[i][2] = __shfl_sync(0xffffffffu, o10, src);
          ao[i][3] = __shfl_sync(0xffffffffu, o11, src);
          aw[i][0] = __shfl_sync(0xffffffffu, w00, src);
          aw[i][1] = __shfl_sync(0xffffffffu, w01, src);
          aw[i][2] = __shfl_sync(0xffffffffu, w10, src);
          aw[i][3] = __shfl_sync(0xffffffffu, w11, src);
          if (!SPLIT) {
#pragma unroll
            for (int c = 0; c < 4; ++c) hw[i][c] = __float2half2_rn(aw[i][c]);
          }
        }
      }
      // (this warpgroup's wgmmas of k-block kb - stages have completed: at most one group is in flight, stages >= 2)
      uint8_t* sa = smem + (size_t)s * STAGE;
      const __half* xc = p.x + kc * DK + piece * 8;
      if (!SPLIT) {
        // fp16 mode: the samples are rounded to fp16 anyway -- blend in packed half2 arithmetic (4 HFMA2 per corner)
        uint4 raw[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int c = 0; c < 4; ++c) raw[i][c] = ldg_nc16(xc + (size_t)ao[i][c] * PS);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          uint4 oh;
          __half2* o2 = reinterpret_cast<__half2*>(&oh);
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const __half2 w2 = hw[i][c];
            const __half2* v2 = reinterpret_cast<const __half2*>(&raw[i][c]);
#pragma unroll
            for (int j = 0; j < 4; ++j) o2[j] = (c == 0) ? __hmul2(w2, v2[j]) : __hfma2(w2, v2[j], o2[j]);
          }
          *reinterpret_cast<uint4*>(sa + sw128_off(gw * 16 + 4 * i + src_sub, piece)) = oh;
        }
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          uint4 rh[4], rl[4];
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const __half* px = xc + (size_t)ao[i][c] * PS;
            rh[c] = ldg_nc16(px);
            rl[c] = ldg_nc16(px + p.C);
          }
          uint4 oh, ol;
          __half2* oh2 = reinterpret_cast<__half2*>(&oh);
          __half2* ol2 = reinterpret_cast<__half2*>(&ol);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float r0 = 0.f, r1 = 0.f;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const float2 f = split2_to_f32(reinterpret_cast<const __half2*>(&rh[c])[j], reinterpret_cast<const __half2*>(&rl[c])[j]);
              r0 = __fmaf_rn(aw[i][c], f.x, r0);
              r1 = __fmaf_rn(aw[i][c], f.y, r1);
            }
            // split2_from_f32 without its clamp (two min/max per element in an issue-bound gather): with sigmoid masks,
            // as in the network, |sample| <= max |x| <= 65504
            oh2[j] = __floats2half2_rn(r0, r1);
            const float2 hf = __half22float2(oh2[j]);
            ol2[j] = lo2_from_f32(r0 - hf.x, r1 - hf.y);
          }
          const uint32_t off = sw128_off(gw * 16 + 4 * i + src_sub, piece);
          *reinterpret_cast<uint4*>(sa + off) = oh;
          *reinterpret_cast<uint4*>(sa + A_TILE + off) = ol;
        }
      }
      fence_proxy_async();   // generic-proxy smem writes -> visible to wgmma (async proxy)
      asm volatile("bar.sync %0, 128;" ::"r"(1 + wgi) : "memory");   // the warpgroup's 64 rows are staged
      mbar_wait(&b_full[s], (uint32_t)(it & 1));
      {
        const uint32_t sa32 = smem_u32(sa) + (uint32_t)wgi * (64u * 128u);
        const uint32_t sb32 = smem_u32(sa) + (uint32_t)(NPL * A_TILE);
        wgmma_fence();
        mma_passes<BN, DK / 16, SPLIT>(
            acc[0], acc[NPL - 1],
            [&](int pl, int k) { return make_sw128_desc(sa32 + (uint32_t)(pl * A_TILE)) + (uint64_t)(2 * k); },
            [&](int pl, int k) { return make_sw128_desc(sb32 + (uint32_t)(pl * B_PLANE)) + (uint64_t)(2 * k); });
        wgmma_commit();
      }
      if (kb > 0) {   // k-block kb - 1 has been read: its weight tile can be refilled
        wgmma_wait<1>();
        if ((tid & 127) == 0) mbar_arrive(&empty_bar[(kb - 1) % stages]);
      }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int pl = 0; pl < NPL; ++pl) fence_regs<BN / 2>(acc[pl]);

    // ===================== epilogue =====================
    const int wq = warp & 3;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = wgi * 64 + wq * 16 + (lane >> 2) + 8 * hh;
      const long long m = m0 + row;
      if (m >= p.M) continue;
      __half* yrow = p.y + m * (long long)(NPL * p.Cout) + n0;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        if (n0 + 8 * j >= p.Cout) break;   // Cout % 8 == 0 is required by the launcher
        const int col = 8 * j + 2 * (lane & 3);
        const int ch = n0 + col;
        const int i = 4 * j + 2 * hh;
        const float a0 = SPLIT ? split_combine(acc[0][i], acc[NPL - 1][i]) : acc[0][i];
        const float a1 = SPLIT ? split_combine(acc[0][i + 1], acc[NPL - 1][i + 1]) : acc[0][i + 1];
        const float v0 = apply_act(scale_bias<SPLIT>(a0, p.out_scale, p.bias ? __ldg(p.bias + ch) : 0.f), p.act);
        const float v1 = apply_act(scale_bias<SPLIT>(a1, p.out_scale, p.bias ? __ldg(p.bias + ch + 1) : 0.f), p.act);
        __half2 hi, lo;
        if (SPLIT) split2_from_f32(v0, v1, hi, lo);
        else hi = f16x2_from_f32(v0, v1);
        *reinterpret_cast<__half2*>(yrow + col) = hi;
        if (SPLIT) *reinterpret_cast<__half2*>(yrow + p.Cout + col) = lo;
      }
    }
  }
}
template <int BN, bool SPLIT>
void launch_dcn_variant(const DcnParams& prm, size_t smem, dim3 grid, cudaStream_t stream) {
  static PerDeviceOnce attr;
  if (attr.first())
    YB_CHECK_CUDA(cudaFuncSetAttribute(dcn_tc_kernel<BN, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(226 * 1024)));
  dcn_tc_kernel<BN, SPLIT><<<grid, DTHREADS, smem, stream>>>(prm);
}

}  // namespace

struct DcnTcPlan {
  DcnParams prm;
  int BN = 128;
  int split = 0;
  size_t smem = 0;
  dim3 grid;
};

bool dcn_tc_supported(int C, int Cout, int dg) {
  return dg >= 1 && C % dg == 0 && (C / dg) % 64 == 0 && Cout % 8 == 0 && Cout >= 8;
}

// w_packed: [Cout][taps*C] fp16, k = tap*C + c  (split: [Cout][hi(taps*C) | lo(taps*C)] of w / out_scale)
DcnTcPlan* dcn_tc_plan_create(const __half* x, const float* om, const __half* w_packed, const float* bias, __half* y, int B,
                              int H, int W, int C, int Ho, int Wo, int Cout, const yb_dcn_params& g, int act,
                              int mask_logits, int split, float out_scale, int bn_override) {
  YB_REQUIRE(dcn_tc_supported(C, Cout, g.deformable_group), "dcn_tc: needs (C / dg) % 64 == 0 and Cout % 8 == 0");
  auto* plan = new DcnTcPlan();
  DcnParams& q = plan->prm;
  memset(&q, 0, sizeof(q));
  plan->split = split ? 1 : 0;
  const int npl = split ? 2 : 1;
  // N tile <= 128: the accumulators of a 64-row half stay within 128 registers per thread in both modes
  int BN = Cout > 64 ? 128 : 64;
  if (bn_override == 64 || bn_override == 128) BN = bn_override;
  plan->BN = BN;
  q.x = x;
  q.om = om;
  q.bias = bias;
  q.y = y;
  q.B = B;
  q.H = H;
  q.W = W;
  q.C = C;
  q.Ho = Ho;
  q.Wo = Wo;
  q.Cout = Cout;
  q.M = (long long)B * Ho * Wo;
  q.g = g;
  q.taps = g.kernel_h * g.kernel_w;
  q.act = act;
  q.mask_logits = mask_logits;
  q.kchunks = C / DK;
  q.gchunks = C / g.deformable_group / DK;
  q.out_scale = split ? out_scale : 1.f;
  const int stage = npl * (A_TILE + BN * DK * 2);
  int stages = std::min(MAX_DSTAGES, (225 * 1024) / stage);
  stages = std::max(2, std::min(stages, q.taps * q.kchunks));   // >= 2: a warpgroup keeps one wgmma group in flight
  q.stages = stages;
  plan->smem = (size_t)stages * stage + 1024;
  plan->grid = dim3((unsigned)((q.M + DM - 1) / DM), (unsigned)ceil_div(Cout, BN), 1);
  const uint64_t KP = (uint64_t)npl * q.taps * C;
  uint64_t dims[3] = {KP, (uint64_t)Cout, 1};
  uint64_t str[2] = {KP * 2, KP * (uint64_t)Cout * 2};
  uint32_t box[3] = {(uint32_t)DK, (uint32_t)BN, 1};
  encode_map_f16(&q.tmW, w_packed, 3, dims, str, box);
  return plan;
}

void dcn_tc_plan_destroy(DcnTcPlan* plan) { delete plan; }

void launch_dcn_tc(const DcnTcPlan* plan, cudaStream_t stream, LaunchCounter* lc) {
  const DcnParams& q = plan->prm;
  if (plan->split) {
    switch (plan->BN) {
      case 128: launch_dcn_variant<128, true>(q, plan->smem, plan->grid, stream); break;
      default: launch_dcn_variant<64, true>(q, plan->smem, plan->grid, stream); break;
    }
  } else {
    switch (plan->BN) {
      case 128: launch_dcn_variant<128, false>(q, plan->smem, plan->grid, stream); break;
      default: launch_dcn_variant<64, false>(q, plan->smem, plan->grid, stream); break;
    }
  }
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

}  // namespace yb
