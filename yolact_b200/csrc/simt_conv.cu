// Generic implicit-GEMM convolution on CUDA cores (fp32 FMA, fp32 accumulation).
//
// Role in the design (DESIGN.md): (1) the whole network in YB_PREC_F32 parity mode, (2) FastMaskIoUNet
// in every mode, (3) on-device second opinion for the tensor-core kernel in tests.
//
// Reference semantics: nn.Conv2d (cross-correlation, zero padding) + folded BatchNorm2d bias
// (backbone.py:37-57) + optional residual add + activation.
//
// GEMM view: M = B*Ho*Wo output pixels, N = Cout, K = KH*KW*Cin with k = (r*KW+s)*Cin + c.
// CTA tile 64(M) x 64(N), K chunk 16, 256 threads, 4x4 outputs per thread.
#include "kernels.cuh"

namespace yb {

namespace {

constexpr int BM = 64, BN = 64, BK = 16, NT = 256;

template <typename TIn, typename TW, typename TOut>
__global__ void __launch_bounds__(NT)
simt_conv_kernel(const TIn* __restrict__ x, const TW* __restrict__ w, const float* __restrict__ bias,
                 const TIn* __restrict__ residual, TOut* __restrict__ y, int B, int H, int W, int Cin,
                 int Ho, int Wo, int Cout, int KH, int KW, int stride, int pad, int act,
                 int x_nchw, int64_t y_batch_stride, int y_pix_stride, int res_after_act) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];

  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const int M = B * Ho * Wo;
  const int K = KH * KW * Cin;

  // A-load role: pixel a_m, 4 consecutive k starting at a_k
  const int a_m = tid >> 2;
  const int a_k = (tid & 3) * 4;
  int a_b = 0, a_ho = 0, a_wo = 0;
  const bool a_valid = (m0 + a_m) < M;
  if (a_valid) {
    int m = m0 + a_m;
    a_wo = m % Wo;
    int t = m / Wo;
    a_ho = t % Ho;
    a_b = t / Ho;
  }
  const int a_hbase = a_ho * stride - pad;
  const int a_wbase = a_wo * stride - pad;

  // B-load role: k row b_k, 4 consecutive n
  const int b_k = tid >> 4;
  const int b_n = (tid & 15) * 4;

  const int ty = tid >> 4, tx = tid & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += BK) {
    // ---- load A chunk
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int k = k0 + a_k + j;
      float v = 0.f;
      if (a_valid && k < K) {
        int tap = k / Cin;
        int c = k - tap * Cin;
        int r = tap / KW;
        int s = tap - r * KW;
        int hi = a_hbase + r;
        int wi = a_wbase + s;
        if (hi >= 0 && hi < H && wi >= 0 && wi < W) {
          size_t idx = x_nchw ? ((size_t)(a_b * Cin + c) * H + hi) * W + wi
                              : ((size_t)(a_b * H + hi) * W + wi) * Cin + c;
          v = to_f32(x[idx]);
        }
      }
      As[a_k + j][a_m] = v;
    }
    // ---- load B chunk
    {
      int k = k0 + b_k;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int n = n0 + b_n + j;
        float v = 0.f;
        if (k < K && n < Cout) v = to_f32(w[(size_t)k * Cout + n]);
        Bs[b_k][b_n + j] = v;
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

  // ---- epilogue
  const int HoWo = Ho * Wo;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int m = m0 + ty * 4 + i;
    if (m >= M) continue;
    int b = m / HoWo;
    int pix = m - b * HoWo;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int n = n0 + tx * 4 + j;
      if (n >= Cout) continue;
      float v = acc[i][j];
      if (bias) v += bias[n];
      if (res_after_act) {
        v = apply_act(v, act);
        if (residual) v += to_f32(residual[(size_t)m * Cout + n]);
      } else {
        if (residual) v += to_f32(residual[(size_t)m * Cout + n]);
        v = apply_act(v, act);
      }
      y[(size_t)b * y_batch_stride + (size_t)pix * y_pix_stride + n] = from_f32<TOut>(v);
    }
  }
}

template <typename TIn, typename TW, typename TOut>
void launch_t(const ConvProblem& p, const void* w, cudaStream_t stream) {
  const int M = p.B * p.Ho * p.Wo;
  dim3 grid(ceil_div(M, BM), ceil_div(p.Cout, BN));
  simt_conv_kernel<TIn, TW, TOut><<<grid, NT, 0, stream>>>(
      (const TIn*)p.x, (const TW*)w, p.bias, (const TIn*)p.residual, (TOut*)p.y, p.B, p.H, p.W,
      p.Cin, p.Ho, p.Wo, p.Cout, p.KH, p.KW, p.stride, p.pad, p.act, p.x_nchw_f32,
      p.y_batch_stride, p.y_pix_stride, p.res_after_act);
  YB_CHECK_LAUNCH();
}

}  // namespace

void launch_simt_conv(const ConvProblem& p, const void* w, int types, cudaStream_t stream,
                      LaunchCounter* lc) {
  YB_REQUIRE(p.x && p.y && w, "simt_conv: null pointer");
  YB_REQUIRE(p.Ho == (p.H + 2 * p.pad - p.KH) / p.stride + 1, "simt_conv: bad Ho");
  YB_REQUIRE(p.Wo == (p.W + 2 * p.pad - p.KW) / p.stride + 1, "simt_conv: bad Wo");
  switch (types) {
    case SIMT_F32:
      launch_t<float, float, float>(p, w, stream);
      break;
    case SIMT_F16:
      YB_REQUIRE(!p.x_nchw_f32, "simt_conv: NCHW input is fp32 only");
      if (p.y_f32)
        launch_t<__half, __half, float>(p, w, stream);
      else
        launch_t<__half, __half, __half>(p, w, stream);
      break;
    default:
      YB_REQUIRE(false, "simt_conv: unknown type combination");
  }
  if (lc) lc->n++;
}

}  // namespace yb
