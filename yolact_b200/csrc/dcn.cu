// DCNv2 modulated deformable convolution (forward): any kh x kw kernel, per-axis stride / padding / dilation,
// deformable groups.
//
// Reference: DCN.forward (external/DCNv2/dcn_v2.py:118-128: out27 -> 18 offsets + sigmoid(9 masks)),
// modulated_deformable_im2col_gpu_kernel (external/DCNv2/src/cuda/dcn_v2_im2col_cuda.cu:125-195),
// dmcn_im2col_bilinear (:25-54), bias + GEMM (src/cuda/dcn_v2_cuda.cu:123-163).
//
// Sampling rule: for output pixel (ho,wo), tap = i*kw + j and the deformable group gr of the input channel:
//     h = ho*stride_h - pad_h + i*dil_h + off[gr][2*tap],  w = wo*stride_w - pad_w + j*dil_w + off[gr][2*tap+1]
//     val = (h > -1 && w > -1 && h < H && w < W) ? bilinear_zero_pad(x, h, w) : 0;  col = val * mask[gr][tap]
// The reference materialises col as [B, C*taps, Ho*Wo] fp32 in HBM and runs two batched SGEMMs.
//  * launch_dcn_simt: fully fused gather + contraction on CUDA cores (fp32 parity mode, the half-precision mode of
//    groups narrower than the tensor-core kernel's 64-channel k-block, and the on-device second opinion for the
//    tensor-core path).
#include <stdlib.h>
#include <string>
#include "kernels.cuh"

namespace yb {

namespace {

struct TapGeom {
  int o00, o01, o10, o11;  // pixel offsets (in pixels) of the 4 corners, -1 when outside
  float w00, w01, w10, w11;
};

// Geometry of one (pixel, tap, deformable group): corner pixel indices + bilinear weights (mask applied by the caller).
// om: the pixel's row of offsets and masks; (i, j) the tap's kernel position.
__device__ __forceinline__ TapGeom tap_geometry(const float* __restrict__ om, int tap, int gr, int taps, int i, int j,
                                                int ho, int wo, int H, int W, const yb_dcn_params& p) {
  const float off_h = om[gr * 2 * taps + 2 * tap], off_w = om[gr * 2 * taps + 2 * tap + 1];
  const float h = __fadd_rn((float)(ho * p.stride_h - p.pad_h + i * p.dilation_h), off_h);
  const float w = __fadd_rn((float)(wo * p.stride_w - p.pad_w + j * p.dilation_w), off_w);
  TapGeom g;
  g.o00 = g.o01 = g.o10 = g.o11 = -1;
  g.w00 = g.w01 = g.w10 = g.w11 = 0.f;
  if (h > -1.f && w > -1.f && h < (float)H && w < (float)W) {
    const int hl = (int)floorf(h), wl = (int)floorf(w);
    const int hh = hl + 1, wh = wl + 1;
    const float lh = __fsub_rn(h, (float)hl), lw = __fsub_rn(w, (float)wl);
    const float uh = __fsub_rn(1.f, lh), uw = __fsub_rn(1.f, lw);
    if (hl >= 0 && wl >= 0) g.o00 = hl * W + wl;
    if (hl >= 0 && wh <= W - 1) g.o01 = hl * W + wh;
    if (hh <= H - 1 && wl >= 0) g.o10 = hh * W + wl;
    if (hh <= H - 1 && wh <= W - 1) g.o11 = hh * W + wh;
    g.w00 = __fmul_rn(uh, uw);
    g.w01 = __fmul_rn(uh, lw);
    g.w10 = __fmul_rn(lh, uw);
    g.w11 = __fmul_rn(lh, lw);
  }
  return g;
}

__device__ __forceinline__ float tap_mask(const float* __restrict__ om, int tap, int gr, int taps, int dg,
                                          int mask_logits) {
  // torch.sigmoid of the mask logits (dcn_v2.py:122); the op-level entry point receives the
  // mask already activated, like dcn_v2_forward does
  const float v = om[2 * dg * taps + gr * taps + tap];
  return mask_logits ? __fdiv_rn(1.f, __fadd_rn(1.f, expf(-v))) : v;
}

constexpr int BM = 64, BN = 64, BK = 16, NT = 256;

template <typename T>
__global__ void __launch_bounds__(NT)
dcn_simt_kernel(const T* __restrict__ x, const float* __restrict__ om, const T* __restrict__ w,
                const float* __restrict__ bias, T* __restrict__ y, int B, int H, int W, int C, int Ho,
                int Wo, int Cout, const yb_dcn_params p, int act, int mask_logits) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int M = B * Ho * Wo;
  const int taps = p.kernel_h * p.kernel_w;
  const int K = taps * C;
  const int dg = p.deformable_group, cg = C / dg;

  const int a_m = tid >> 2, a_k = (tid & 3) * 4;
  const bool a_valid = (m0 + a_m) < M;
  int a_b = 0, a_ho = 0, a_wo = 0;
  if (a_valid) {
    int m = m0 + a_m;
    a_wo = m % Wo;
    int t = m / Wo;
    a_ho = t % Ho;
    a_b = t / Ho;
  }
  const float* a_om = om + (size_t)(m0 + a_m) * (3 * dg * taps);
  const T* a_x = x + (size_t)a_b * H * W * C;
  const int b_k = tid >> 4, b_n = (tid & 15) * 4;
  const int ty = tid >> 4, tx = tid & 15;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  // (tap, channel) of this thread's first column k = k0 + a_k, advanced with k0: a chunk may straddle taps and groups
  // (any C), so the geometry is looked up per column and recomputed when its (tap, group) changes
  int k_tap = 0, k_c = a_k;
  while (k_c >= C) k_c -= C, ++k_tap;
  int cur_key = -1;
  TapGeom g;
  float msk = 0.f;
  for (int k0 = 0; k0 < K; k0 += BK) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int c = k_c + j, tap = k_tap;
      while (c >= C) c -= C, ++tap;
      float v = 0.f;
      if (a_valid && tap < taps) {
        const int gr = dg == 1 ? 0 : c / cg;
        const int key = tap * dg + gr;
        if (key != cur_key) {
          const int ti = tap / p.kernel_w;
          g = tap_geometry(a_om, tap, gr, taps, ti, tap - ti * p.kernel_w, a_ho, a_wo, H, W, p);
          msk = tap_mask(a_om, tap, gr, taps, dg, mask_logits);
          cur_key = key;
        }
        float v1 = g.o00 >= 0 ? to_f32(a_x[(size_t)g.o00 * C + c]) : 0.f;
        float v2 = g.o01 >= 0 ? to_f32(a_x[(size_t)g.o01 * C + c]) : 0.f;
        float v3 = g.o10 >= 0 ? to_f32(a_x[(size_t)g.o10 * C + c]) : 0.f;
        float v4 = g.o11 >= 0 ? to_f32(a_x[(size_t)g.o11 * C + c]) : 0.f;
        // (w1*v1 + w2*v2 + w3*v3 + w4*v4) * mask, left to right (im2col_cuda.cu:50-53,189)
        float val = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(g.w00, v1), __fmul_rn(g.w01, v2)),
                                        __fmul_rn(g.w10, v3)),
                              __fmul_rn(g.w11, v4));
        v = __fmul_rn(val, msk);
      }
      As[a_k + j][a_m] = v;
    }
    k_c += BK;
    while (k_c >= C) k_c -= C, ++k_tap;
    {
      const int k = k0 + b_k;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = n0 + b_n + j;
        Bs[b_k][b_n + j] = (k < K && n < Cout) ? to_f32(w[(size_t)k * Cout + n]) : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= Cout) continue;
      float v = acc[i][j];
      if (bias) v += bias[n];
      y[(size_t)m * Cout + n] = from_f32<T>(apply_act(v, act));
    }
  }
}

}  // namespace

template <typename T>
void launch_dcn_simt(const T* x, const float* om, const T* w, const float* bias, T* y, int B, int H, int W, int C,
                     int Ho, int Wo, int Cout, const yb_dcn_params& g, int act, int mask_logits, cudaStream_t stream,
                     LaunchCounter* lc) {
  YB_REQUIRE(g.deformable_group >= 1 && C % g.deformable_group == 0, "dcn: C must be a multiple of deformable_group");
  const int M = B * Ho * Wo;
  dim3 grid(ceil_div(M, BM), ceil_div(Cout, BN));
  dcn_simt_kernel<T><<<grid, NT, 0, stream>>>(x, om, w, bias, y, B, H, W, C, Ho, Wo, Cout, g, act, mask_logits);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}
template void launch_dcn_simt<float>(const float*, const float*, const float*, const float*, float*, int, int, int,
                                     int, int, int, int, const yb_dcn_params&, int, int, cudaStream_t, LaunchCounter*);
template void launch_dcn_simt<__half>(const __half*, const float*, const __half*, const float*, __half*, int, int,
                                      int, int, int, int, int, const yb_dcn_params&, int, int, cudaStream_t,
                                      LaunchCounter*);

}  // namespace yb
