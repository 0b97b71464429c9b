// DCNv2 modulated deformable convolution (forward), deformable_groups = 1.
//
// Reference: DCN.forward (external/DCNv2/dcn_v2.py:118-128: out27 -> 18 offsets + sigmoid(9 masks)),
// modulated_deformable_im2col_gpu_kernel (external/DCNv2/src/cuda/dcn_v2_im2col_cuda.cu:125-195),
// dmcn_im2col_bilinear (:25-54), bias + GEMM (src/cuda/dcn_v2_cuda.cu:123-163).
//
// Sampling rule: for output pixel (ho,wo) and tap k=(i,j):
//     h = ho*stride - pad + i*dil + off[2k],  w = wo*stride - pad + j*dil + off[2k+1]
//     val = (h > -1 && w > -1 && h < H && w < W) ? bilinear_zero_pad(x, h, w) : 0;  col = val * mask[k]
// The reference materialises col as [B, C*9, Ho*Wo] fp32 in HBM and runs two batched SGEMMs.
//  * launch_dcn_simt: fully fused gather + contraction on CUDA cores (fp32 parity mode, and the
//    on-device second opinion for the tensor-core path).
//  * launch_dcn_gather_f16: gather to fp16 NHWC columns [B,Ho,Wo,9*C] (2 B/element instead of
//    4, channel-contiguous 16-byte stores) consumed by the tensor-core kernel as a 1x1 conv, K = 9*C.
//    Kept behind YB_DCN_FUSED=0 as the A/B partner of the fused kernel (dcn_tc.cu), which is the default: one launch,
//    no column buffer.
#include <stdlib.h>
#include <string>
#include "kernels.cuh"

namespace yb {

namespace {

struct TapGeom {
  int o00, o01, o10, o11;  // pixel offsets (in pixels) of the 4 corners, -1 when outside
  float w00, w01, w10, w11;
};

// Geometry of one (pixel, tap): corner pixel indices + bilinear weights (mask applied by the caller).
__device__ __forceinline__ TapGeom tap_geometry(const float* __restrict__ om, int tap, int ho, int wo,
                                                int H, int W, int stride, int pad, int dil) {
  const int i = tap / 3, j = tap - i * 3;
  const float off_h = om[2 * tap], off_w = om[2 * tap + 1];
  const float h = __fadd_rn((float)(ho * stride - pad + i * dil), off_h);
  const float w = __fadd_rn((float)(wo * stride - pad + j * dil), off_w);
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

__device__ __forceinline__ float tap_mask(const float* __restrict__ om, int tap, int mask_logits) {
  // torch.sigmoid of the 9 mask logits (dcn_v2.py:122); the op-level entry point receives the
  // mask already activated, like dcn_v2_forward does
  const float v = om[18 + tap];
  return mask_logits ? __fdiv_rn(1.f, __fadd_rn(1.f, expf(-v))) : v;
}

constexpr int BM = 64, BN = 64, BK = 16, NT = 256;

template <typename T>
__global__ void __launch_bounds__(NT)
dcn_simt_kernel(const T* __restrict__ x, const float* __restrict__ om, const T* __restrict__ w,
                const float* __restrict__ bias, T* __restrict__ y, int B, int H, int W, int C, int Ho,
                int Wo, int Cout, int stride, int pad, int dil, int act, int mask_logits) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int M = B * Ho * Wo;
  const int K = 9 * C;

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
  const float* a_om = om + (size_t)(m0 + a_m) * 27;
  const T* a_x = x + (size_t)a_b * H * W * C;
  const int b_k = tid >> 4, b_n = (tid & 15) * 4;
  const int ty = tid >> 4, tx = tid & 15;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  int cur_tap = -1;
  TapGeom g;
  float msk = 0.f;
  for (int k0 = 0; k0 < K; k0 += BK) {
    const int tap = k0 / C;  // C % 16 == 0: a chunk never straddles taps
    const int c0 = k0 - tap * C;
    if (a_valid && tap != cur_tap) {
      g = tap_geometry(a_om, tap, a_ho, a_wo, H, W, stride, pad, dil);
      msk = tap_mask(a_om, tap, mask_logits);
      cur_tap = tap;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float v = 0.f;
      if (a_valid) {
        const int c = c0 + a_k + j;
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

// one thread = (pixel, tap, 8 channels).  split: x is [hi(C) | lo(C)] per pixel (sample = hi + lo) and the columns are
// written as [hi(9C) | lo(9C)] per output pixel (YB_PREC_F16X3).
__global__ void dcn_gather_f16_kernel(const __half* __restrict__ x, const float* __restrict__ om,
                                      __half* __restrict__ cols, int B, int H, int W, int C, int Ho,
                                      int Wo, int stride, int pad, int dil, int mask_logits, int split) {
  const int CV = C / 8;
  const int PS = split ? 2 * C : C;
  const int64_t total = (int64_t)B * Ho * Wo * 9 * CV;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int cv = (int)(idx % CV);
    int64_t t = idx / CV;
    const int tap = (int)(t % 9);
    const int64_t m = t / 9;
    const int wo = (int)(m % Wo);
    const int64_t t2 = m / Wo;
    const int ho = (int)(t2 % Ho);
    const int b = (int)(t2 / Ho);
    const float* pom = om + m * 27;
    const TapGeom g = tap_geometry(pom, tap, ho, wo, H, W, stride, pad, dil);
    const float msk = tap_mask(pom, tap, mask_logits);
    const __half* xb = x + (size_t)b * H * W * PS + cv * 8;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    auto corner = [&](int o, float wgt) {
      if (o < 0) return;
      uint4 raw = *reinterpret_cast<const uint4*>(xb + (size_t)o * PS);
      const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
      float f8[8];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 f = __half22float2(h2[j]);
        f8[2 * j] = f.x;
        f8[2 * j + 1] = f.y;
      }
      if (split) {
        uint4 rawl = *reinterpret_cast<const uint4*>(xb + (size_t)o * PS + C);
        const __half2* l2 = reinterpret_cast<const __half2*>(&rawl);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 f = lo2_to_f32(l2[j]);   // lo plane: residual * 2^11
          f8[2 * j] += f.x;
          f8[2 * j + 1] += f.y;
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = fmaf(wgt, f8[j], acc[j]);
    };
    corner(g.o00, g.w00);
    corner(g.o01, g.w01);
    corner(g.o10, g.w10);
    corner(g.o11, g.w11);
    uint4 outv, outl;
    __half2* o2 = reinterpret_cast<__half2*>(&outv);
    __half2* ol2 = reinterpret_cast<__half2*>(&outl);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float v0 = acc[2 * j] * msk, v1 = acc[2 * j + 1] * msk;
      o2[j] = __halves2half2(from_f32<__half>(v0), from_f32<__half>(v1));
      if (split) {
        const float2 hf = __half22float2(o2[j]);
        ol2[j] = lo2_from_f32(fabsf(v0) > 65504.f ? 0.f : v0 - hf.x, fabsf(v1) > 65504.f ? 0.f : v1 - hf.y);   // lo' = residual * 2^11
      }
    }
    __half* cp = cols + (size_t)m * 9 * PS + (size_t)tap * C + cv * 8;
    *reinterpret_cast<uint4*>(cp) = outv;
    if (split) *reinterpret_cast<uint4*>(cp + 9 * C) = outl;
  }
}


}  // namespace

template <typename T>
void launch_dcn_simt(const T* x, const float* om, const T* w, const float* bias, T* y, int B, int H,
                     int W, int C, int Ho, int Wo, int Cout, int stride, int pad, int dil, int act,
                     int mask_logits, cudaStream_t stream, LaunchCounter* lc) {
  YB_REQUIRE(C % 16 == 0, "dcn: C must be a multiple of 16");
  const int M = B * Ho * Wo;
  dim3 grid(ceil_div(M, BM), ceil_div(Cout, BN));
  dcn_simt_kernel<T><<<grid, NT, 0, stream>>>(x, om, w, bias, y, B, H, W, C, Ho, Wo, Cout, stride, pad,
                                             dil, act, mask_logits);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}
template void launch_dcn_simt<float>(const float*, const float*, const float*, const float*, float*,
                                     int, int, int, int, int, int, int, int, int, int, int, int,
                                     cudaStream_t, LaunchCounter*);
template void launch_dcn_simt<__half>(const __half*, const float*, const __half*, const float*,
                                      __half*, int, int, int, int, int, int, int, int, int, int, int, int,
                                      cudaStream_t, LaunchCounter*);

void launch_dcn_gather_f16(const __half* x, const float* om, __half* cols, int B, int H, int W,
                           int C, int Ho, int Wo, int stride, int pad, int dil, int mask_logits,
                           cudaStream_t stream, LaunchCounter* lc, int split) {
  YB_REQUIRE(C % 8 == 0, "dcn gather: C must be a multiple of 8");
  const int64_t total = (int64_t)B * Ho * Wo * 9 * (C / 8);
  int64_t g = (total + 255) / 256;
  if (g > 132 * 32) g = 132 * 32;
  dcn_gather_f16_kernel<<<(unsigned)g, 256, 0, stream>>>(x, om, cols, B, H, W, C, Ho, Wo, stride, pad, dil, mask_logits, split);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

}  // namespace yb
