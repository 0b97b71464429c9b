// HBM-bound pointwise / resampling kernels of the conv stack.  All NHWC, 16-byte vectorised over
// the channel dimension where the channel count allows it.
#include "kernels.cuh"

namespace yb {

namespace {

template <typename T>
struct Vec16 {
  uint4 raw;
};

template <typename T>
__device__ __forceinline__ void unpack(const uint4& r, float* f);
template <>
__device__ __forceinline__ void unpack<float>(const uint4& r, float* f) {
  f[0] = __uint_as_float(r.x);
  f[1] = __uint_as_float(r.y);
  f[2] = __uint_as_float(r.z);
  f[3] = __uint_as_float(r.w);
}
template <>
__device__ __forceinline__ void unpack<__half>(const uint4& r, float* f) {
  const __half2* h = reinterpret_cast<const __half2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __half22float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
template <typename T>
__device__ __forceinline__ uint4 pack(const float* f);
template <>
__device__ __forceinline__ uint4 pack<float>(const float* f) {
  return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]),
                    __float_as_uint(f[3]));
}
template <>
__device__ __forceinline__ uint4 pack<__half>(const float* f) {
  uint4 r;
  __half2* h = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __halves2half2(from_f32<__half>(f[2 * i]), from_f32<__half>(f[2 * i + 1]));
  return r;
}

// lo-plane element access for the scalar layout kernels (split tensors exist for T = __half only)
__device__ __forceinline__ float lo_of(float) { return 0.f; }
__device__ __forceinline__ float lo_of(__half h) { return lo_to_f32(h); }
template <typename T>
__device__ __forceinline__ T lo_make(float r);
template <>
__device__ __forceinline__ float lo_make<float>(float r) {
  return r;
}
template <>
__device__ __forceinline__ __half lo_make<__half>(float r) {
  return lo_from_f32(r);
}

// One 16-byte channel vector of a pixel -> floats.  `px` points at the pixel's first element; split (fp16 only):
// the pixel is [hi(C) | lo(C)] and the value is hi + lo (YB_PREC_F16X3).
template <typename T>
__device__ __forceinline__ void load_vec(const T* px, int C, int cv, int split, float* f) {
  constexpr int V = DType<T>::kVec;
  unpack<T>(*reinterpret_cast<const uint4*>(px + cv * V), f);
  if (sizeof(T) == 2 && split) {   // lo plane: residual * 2^11
    const uint4 rl = *reinterpret_cast<const uint4*>(px + C + cv * V);
    const __half2* l2 = reinterpret_cast<const __half2*>(&rl);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 t = lo2_to_f32(l2[j]);
      f[(2 * j) % V] += t.x;
      f[(2 * j + 1) % V] += t.y;
    }
  }
}
template <typename T>
__device__ __forceinline__ void store_vec(T* px, int C, int cv, int split, const float* f) {
  constexpr int V = DType<T>::kVec;
  const uint4 hi = pack<T>(f);
  *reinterpret_cast<uint4*>(px + cv * V) = hi;
  if (sizeof(T) == 2 && split) {
    float h[V], l[8];
    unpack<T>(hi, h);
#pragma unroll
    for (int j = 0; j < 8; ++j) l[j] = fabsf(f[j % V]) > 65504.f ? 0.f : f[j % V] - h[j % V];
    uint4 lo;
    __half2* l2 = reinterpret_cast<__half2*>(&lo);
#pragma unroll
    for (int j = 0; j < 4; ++j) l2[j] = lo2_from_f32(l[2 * j], l[2 * j + 1]);
    *reinterpret_cast<uint4*>(px + C + cv * V) = lo;
  }
}

// ---- 3x3/s2/p1 max pool (backbone.py:80).  Padding acts as -inf (PyTorch semantics). ----------
template <typename T>
__global__ void maxpool3x3s2_kernel(const T* __restrict__ x, T* __restrict__ y, int B, int H, int W,
                                    int C, int Ho, int Wo, int split) {
  constexpr int V = DType<T>::kVec;
  const int CV = C / V;
  const int PS = split ? 2 * C : C;   // elements per pixel
  const int64_t total = (int64_t)B * Ho * Wo * CV;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int cv = (int)(i % CV);
    int64_t t = i / CV;
    int wo = (int)(t % Wo);
    t /= Wo;
    int ho = (int)(t % Ho);
    int b = (int)(t / Ho);
    float m[V];
#pragma unroll
    for (int j = 0; j < V; ++j) m[j] = -INFINITY;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      int hi = ho * 2 - 1 + r;
      if (hi < 0 || hi >= H) continue;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        int wi = wo * 2 - 1 + s;
        if (wi < 0 || wi >= W) continue;
        float f[V];
        load_vec<T>(x + (((int64_t)b * H + hi) * W + wi) * PS, C, cv, split, f);
#pragma unroll
        for (int j = 0; j < V; ++j) m[j] = fmaxf(m[j], f[j]);
      }
    }
    store_vec<T>(y + (((int64_t)b * Ho + ho) * Wo + wo) * PS, C, cv, split, m);
  }
}

// ---- bilinear resize, align_corners=False (ATen upsample_bilinear2d) ----------------------------
// src = max(scale*(dst+0.5)-0.5, 0); lo = floor(src); hi = lo + (lo < in-1); lam = src - lo
// value = l0h*(l0w*p00 + l1w*p01) + l1h*(l0w*p10 + l1w*p11)      (SURVEY.md Appendix D.12)
template <typename T>
__global__ void upsample_bilinear_kernel(const T* __restrict__ x, const T* __restrict__ add,
                                         T* __restrict__ y, int B, int H, int W, int C, int Ho,
                                         int Wo, float scale_h, float scale_w, int relu, int split) {
  constexpr int V = DType<T>::kVec;
  const int CV = C / V;
  const int PS = split ? 2 * C : C;
  const int64_t total = (int64_t)B * Ho * Wo * CV;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int cv = (int)(i % CV);
    int64_t t = i / CV;
    int wo = (int)(t % Wo);
    t /= Wo;
    int ho = (int)(t % Ho);
    int b = (int)(t / Ho);
    float sh = fmaxf(__fsub_rn(__fmul_rn(scale_h, (float)ho + 0.5f), 0.5f), 0.f);
    float sw = fmaxf(__fsub_rn(__fmul_rn(scale_w, (float)wo + 0.5f), 0.5f), 0.f);
    int h0 = (int)sh, w0 = (int)sw;
    int h1 = h0 + (h0 < H - 1 ? 1 : 0);
    int w1 = w0 + (w0 < W - 1 ? 1 : 0);
    float l1h = sh - (float)h0, l1w = sw - (float)w0;
    float l0h = 1.f - l1h, l0w = 1.f - l1w;
    const T* base = x + (int64_t)b * H * W * PS;
    float p00[V], p01[V], p10[V], p11[V], o[V];
    load_vec<T>(base + ((int64_t)h0 * W + w0) * PS, C, cv, split, p00);
    load_vec<T>(base + ((int64_t)h0 * W + w1) * PS, C, cv, split, p01);
    load_vec<T>(base + ((int64_t)h1 * W + w0) * PS, C, cv, split, p10);
    load_vec<T>(base + ((int64_t)h1 * W + w1) * PS, C, cv, split, p11);
    const int64_t opix = (((int64_t)b * Ho + ho) * Wo + wo) * PS;
    float a[V];
    if (add) load_vec<T>(add + opix, C, cv, split, a);
#pragma unroll
    for (int j = 0; j < V; ++j) {
      float top = __fadd_rn(__fmul_rn(l0w, p00[j]), __fmul_rn(l1w, p01[j]));
      float bot = __fadd_rn(__fmul_rn(l0w, p10[j]), __fmul_rn(l1w, p11[j]));
      float v = __fadd_rn(__fmul_rn(l0h, top), __fmul_rn(l1h, bot));
      if (add) v = __fadd_rn(v, a[j]);
      if (relu) v = fmaxf(v, 0.f);
      o[j] = v;
    }
    store_vec<T>(y + opix, C, cv, split, o);
  }
}

// ---- layout conversion (tile transpose through shared memory) -----------------------------------
// NHWC(T) [B, HW, C] -> NCHW fp32 [B, C, HW]
template <typename T>
__global__ void nhwc_to_nchw_kernel(const T* __restrict__ x, float* __restrict__ y, int HW, int C, int split) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int PS = split ? 2 * C : C;
  const T* xb = x + (int64_t)b * HW * PS;
  float* yb_ = y + (int64_t)b * HW * C;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int p = p0 + i, c = c0 + threadIdx.x;
    float v = 0.f;
    if (p < HW && c < C) {
      v = to_f32(xb[(int64_t)p * PS + c]);
      if (split) v += lo_of(xb[(int64_t)p * PS + C + c]);
    }
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, p = p0 + threadIdx.x;
    if (c < C && p < HW) yb_[(int64_t)c * HW + p] = tile[threadIdx.x][i];
  }
}
// NCHW fp32 [B, C, HW] -> NHWC(T) [B, HW, C]
template <typename T>
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, T* __restrict__ y, int HW, int C, int split) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int PS = split ? 2 * C : C;
  const float* xb = x + (int64_t)b * HW * C;
  T* yb_ = y + (int64_t)b * HW * PS;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, p = p0 + threadIdx.x;
    tile[i][threadIdx.x] = (p < HW && c < C) ? xb[(int64_t)c * HW + p] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int p = p0 + i, c = c0 + threadIdx.x;
    if (c < C && p < HW) {
      const float v = tile[threadIdx.x][i];
      const T hi = from_f32<T>(v);
      yb_[(int64_t)p * PS + c] = hi;
      if (split) yb_[(int64_t)p * PS + C + c] = lo_make<T>(fabsf(v) > 65504.f ? 0.f : v - to_f32(hi));
    }
  }
}

// ---- row softmax (yolact.py:674), one warp per row, cols <= 1024 ---------------------------------
__global__ void softmax_rows_kernel(const float* __restrict__ in, float* __restrict__ out,
                                    int64_t rows, int cols) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (row >= rows) return;
  const float* r = in + row * cols;
  float m = -INFINITY;
  for (int c = lane; c < cols; c += 32) m = fmaxf(m, r[c]);
#pragma unroll
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float s = 0.f;
  for (int c = lane; c < cols; c += 32) s += expf(r[c] - m);
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  float* w = out + row * cols;
  for (int c = lane; c < cols; c += 32) w[c] = __fdiv_rn(expf(r[c] - m), s);
}

__global__ void fill_u32_kernel(uint32_t* p, uint32_t v, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    p[i] = v;
}

inline int grid_for(int64_t total, int block) {
  int64_t g = (total + block - 1) / block;
  const int64_t cap = 132 * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

template <typename T>
void launch_maxpool3x3s2(const T* x, T* y, int B, int H, int W, int C, int Ho, int Wo,
                         cudaStream_t stream, LaunchCounter* lc, int split) {
  YB_REQUIRE(C % DType<T>::kVec == 0, "maxpool: C must be a multiple of the vector width");
  YB_REQUIRE(!split || sizeof(T) == 2, "split activations are fp16 pairs");
  int64_t total = (int64_t)B * Ho * Wo * (C / DType<T>::kVec);
  maxpool3x3s2_kernel<T><<<grid_for(total, 256), 256, 0, stream>>>(x, y, B, H, W, C, Ho, Wo, split);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}
template void launch_maxpool3x3s2<float>(const float*, float*, int, int, int, int, int, int,
                                         cudaStream_t, LaunchCounter*, int);
template void launch_maxpool3x3s2<__half>(const __half*, __half*, int, int, int, int, int, int,
                                          cudaStream_t, LaunchCounter*, int);

template <typename T>
void launch_upsample_bilinear(const T* x, const T* add, T* y, int B, int H, int W, int C, int Ho,
                              int Wo, float scale_h, float scale_w, int relu, cudaStream_t stream,
                              LaunchCounter* lc, int split) {
  YB_REQUIRE(C % DType<T>::kVec == 0, "upsample: C must be a multiple of the vector width");
  YB_REQUIRE(!split || sizeof(T) == 2, "split activations are fp16 pairs");
  int64_t total = (int64_t)B * Ho * Wo * (C / DType<T>::kVec);
  upsample_bilinear_kernel<T><<<grid_for(total, 256), 256, 0, stream>>>(x, add, y, B, H, W, C, Ho, Wo,
                                                                       scale_h, scale_w, relu, split);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}
template void launch_upsample_bilinear<float>(const float*, const float*, float*, int, int, int, int,
                                              int, int, float, float, int, cudaStream_t,
                                              LaunchCounter*, int);
template void launch_upsample_bilinear<__half>(const __half*, const __half*, __half*, int, int, int,
                                               int, int, int, float, float, int, cudaStream_t,
                                               LaunchCounter*, int);

template <typename T>
void launch_nhwc_to_nchw_f32(const T* x, float* y, int B, int H, int W, int C, cudaStream_t stream,
                             LaunchCounter* lc, int split) {
  int HW = H * W;
  dim3 grid(ceil_div(HW, 32), ceil_div(C, 32), B), block(32, 8);
  nhwc_to_nchw_kernel<T><<<grid, block, 0, stream>>>(x, y, HW, C, split);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}
template void launch_nhwc_to_nchw_f32<float>(const float*, float*, int, int, int, int, cudaStream_t,
                                             LaunchCounter*, int);
template void launch_nhwc_to_nchw_f32<__half>(const __half*, float*, int, int, int, int,
                                              cudaStream_t, LaunchCounter*, int);

template <typename T>
void launch_nchw_f32_to_nhwc(const float* x, T* y, int B, int C, int H, int W, cudaStream_t stream,
                             LaunchCounter* lc, int split) {
  int HW = H * W;
  dim3 grid(ceil_div(HW, 32), ceil_div(C, 32), B), block(32, 8);
  nchw_to_nhwc_kernel<T><<<grid, block, 0, stream>>>(x, y, HW, C, split);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}
template void launch_nchw_f32_to_nhwc<float>(const float*, float*, int, int, int, int, cudaStream_t,
                                             LaunchCounter*, int);
template void launch_nchw_f32_to_nhwc<__half>(const float*, __half*, int, int, int, int,
                                              cudaStream_t, LaunchCounter*, int);

void launch_softmax_rows(const float* in, float* out, int64_t rows, int cols, cudaStream_t stream,
                         LaunchCounter* lc) {
  if (rows == 0) return;
  int64_t threads = rows * 32;
  softmax_rows_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(in, out, rows, cols);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

void launch_fill_u32(uint32_t* p, uint32_t v, int64_t n, cudaStream_t stream, LaunchCounter* lc) {
  if (n == 0) return;
  fill_u32_kernel<<<grid_for(n, 256), 256, 0, stream>>>(p, v, n);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

}  // namespace yb
