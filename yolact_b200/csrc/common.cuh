// Shared helpers for the yolact_b200 CUDA sources (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <stdexcept>

#include "../../include/yolact_b200.h"

namespace yb {

// ---- error plumbing -------------------------------------------------------------------------
struct Error : public std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

void set_last_error(const std::string& msg);

#define YB_CHECK_CUDA(expr)                                                                    \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      throw ::yb::Error(YB_ERR_CUDA, std::string(#expr) + " failed: " + cudaGetErrorString(_e) + \
                                         " (" + __FILE__ + ":" + std::to_string(__LINE__) + ")"); \
    }                                                                                          \
  } while (0)

#define YB_REQUIRE(cond, msg)                                                                  \
  do {                                                                                         \
    if (!(cond)) {                                                                             \
      throw ::yb::Error(YB_ERR_INVALID, std::string(msg) + " [" #cond "] (" + __FILE__ + ":" + \
                                            std::to_string(__LINE__) + ")");                   \
    }                                                                                          \
  } while (0)

// Checks the launch itself (not completion); cheap and capture-safe.
#define YB_CHECK_LAUNCH() YB_CHECK_CUDA(cudaGetLastError())

// ---- enums shared by kernels ----------------------------------------------------------------
enum ActKind : int { ACT_NONE = 0, ACT_RELU = 1, ACT_TANH = 2, ACT_LEAKY = 3 };

template <typename T>
struct DType;
template <>
struct DType<float> {
  static constexpr int kVec = 4;  // elements per 16-byte vector
};
template <>
struct DType<__half> {
  static constexpr int kVec = 8;
};

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
// from_f32, lo_from_f32 and split_f32 are also the host weight packer's encoders (engine.cu pack_weights)
template <typename T>
__host__ __device__ __forceinline__ T from_f32(float v);
template <>
__host__ __device__ __forceinline__ float from_f32<float>(float v) {
  return v;
}
template <>
__host__ __device__ __forceinline__ __half from_f32<__half>(float v) {
  // saturate instead of producing inf: fp16 max is 65504
  v = fminf(fmaxf(v, -65504.f), 65504.f);
  return __float2half_rn(v);
}

// Split-precision operands (YB_PREC_F16X3): a value v is stored as a pair of fp16 numbers (hi, lo') with
//     hi = rn(v),   lo' = rn((v - hi) * 2^11),   v ~= hi + lo' * 2^-11        (22 significand bits).
// The lo plane is kept PRE-SCALED by 2^11: the unscaled residual (<= 2^-12 |v|) is an fp16 SUBNORMAL for every
// |v| < 0.25 and the tensor core flushes fp16 subnormal inputs to zero, and the fp16 MMA takes both operands in the
// same 16-bit format (no bf16 A with an fp16 B), so a wider-exponent lo format is not an option.  The kernels therefore
// accumulate the two cross terms lo'_a * hi_w + hi_a * lo'_w in a SECOND fp32 accumulator and combine
// acc_hi + 2^-11 * acc_lo  in the epilogue.
// Weights are additionally multiplied by a per-layer power of two (engine.cu split_exponent) so that hi uses the upper
// fp16 exponent range.  A pixel of a split NHWC tensor is [hi(C) | lo'(C)], i.e. 2*C halfs.
// The pair is encoded (split_f32, split2_from_f32) and decoded (split_to_f32, split2_to_f32) only here; the three MMA
// passes and the accumulator combine are tc_common.cuh mma_passes and split_combine.
#define YB_LO_SCALE 2048.f
#define YB_LO_INV 4.8828125e-4f   /* 2^-11 */
__host__ __device__ __forceinline__ __half lo_from_f32(float r) { return __float2half_rn(r * YB_LO_SCALE); }
__host__ __device__ __forceinline__ float lo_to_f32(__half h) { return __half2float(h) * YB_LO_INV; }
__host__ __device__ __forceinline__ __half2 lo2_from_f32(float r0, float r1) {
  return __floats2half2_rn(r0 * YB_LO_SCALE, r1 * YB_LO_SCALE);
}
__host__ __device__ __forceinline__ float2 lo2_to_f32(__half2 h) {
  const float2 f = __half22float2(h);
  return make_float2(f.x * YB_LO_INV, f.y * YB_LO_INV);
}
// saturating fp16 pair: +-65504 instead of inf
__host__ __device__ __forceinline__ __half2 f16x2_from_f32(float a, float b) {
  a = fminf(fmaxf(a, -65504.f), 65504.f);
  b = fminf(fmaxf(b, -65504.f), 65504.f);
  return __floats2half2_rn(a, b);
}
// (hi saturates at +-65504; the residual is taken against the clamped value, so a saturated element gets lo = 0 and
// hi + lo stays finite)
__host__ __device__ __forceinline__ void split_f32(float v, __half& hi, __half& lo) {
  const float c = fminf(fmaxf(v, -65504.f), 65504.f);
  hi = __float2half_rn(c);
  lo = lo_from_f32(c - __half2float(hi));
}
// split_f32 of two lanes
__host__ __device__ __forceinline__ void split2_from_f32(float v0, float v1, __half2& hi, __half2& lo) {
  hi = f16x2_from_f32(v0, v1);
  const float2 hf = __half22float2(hi);
  const float c0 = fminf(fmaxf(v0, -65504.f), 65504.f), c1 = fminf(fmaxf(v1, -65504.f), 65504.f);
  lo = lo2_from_f32(c0 - hf.x, c1 - hf.y);
}
__host__ __device__ __forceinline__ float split_to_f32(__half hi, __half lo) { return __half2float(hi) + lo_to_f32(lo); }
__host__ __device__ __forceinline__ float2 split2_to_f32(__half2 hi, __half2 lo) {
  const float2 h = __half22float2(hi), l = lo2_to_f32(lo);
  return make_float2(h.x + l.x, h.y + l.y);
}

// activation with a compile-time selector: the epilogue loops use it directly, a runtime selector goes through apply_act
template <int ACT>
__device__ __forceinline__ float act_t(float v) {
  if (ACT == ACT_RELU) return fmaxf(v, 0.f);
  if (ACT == ACT_LEAKY) return v > 0.f ? v : 0.1f * v;
  if (ACT == ACT_TANH) return tanhf(v);
  return v;
}
__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act) {
    case ACT_RELU: return act_t<ACT_RELU>(v);
    case ACT_TANH: return act_t<ACT_TANH>(v);
    case ACT_LEAKY: return act_t<ACT_LEAKY>(v);
    default: return v;
  }
}

// ---- FastBaseTransform's per-pixel arithmetic (utils/augmentations.py:616-658) ---------------------------------------
// The only definition: evalops.cu's fast_base_transform_kernel writes it to an NCHW fp32 tensor, the frame-list stem
// (stem_tc.cu) computes it inside its loader, so both give the network bit for bit the same input.
struct XformAffine {   // BGR order
  float mean[3];
  float stdv[3];
};
// One axis of ATen's area_pixel_compute_source_index + guard_index_and_lambda (UpSample.h), align_corners=False:
// output coordinate o reads source taps i0 and i1 with weights 1 - l1 and l1.  scale = (float)in_n / (float)out_n.
struct XformTap {
  int i0, i1;
  float l1;
};
__device__ __forceinline__ XformTap xform_tap(int o, int out_n, int in_n, float scale) {
  XformTap t{o, o, 0.f};
  if (out_n != in_n) {
    const float s = fmaxf(__fsub_rn(__fmul_rn(scale, (float)o + 0.5f), 0.5f), 0.f);
    t.i0 = min((int)s, in_n - 1);
    t.i1 = t.i0 + (t.i0 < in_n - 1 ? 1 : 0);
    t.l1 = fminf(fmaxf(s - (float)t.i0, 0.f), 1.f);
  }
  return t;
}
__device__ __forceinline__ float xform_load(const uint8_t* p) { return (float)*p; }
__device__ __forceinline__ float xform_load(const float* p) { return *p; }
// One output pixel of an HWC BGR image of width W: four-tap blend, then (v - mean) / std | v - mean | v / 255 | v
// (yb_transform_mode), written to rgb[] in RGB order.
template <typename TIn>
__device__ __forceinline__ void xform_pixel(const TIn* img, int W, XformTap th, XformTap tw, int mode,
                                            const XformAffine& aff, float rgb[3]) {
  const float l0h = 1.f - th.l1, l0w = 1.f - tw.l1;
  const TIn* p00 = img + ((size_t)th.i0 * W + tw.i0) * 3;
  const TIn* p01 = img + ((size_t)th.i0 * W + tw.i1) * 3;
  const TIn* p10 = img + ((size_t)th.i1 * W + tw.i0) * 3;
  const TIn* p11 = img + ((size_t)th.i1 * W + tw.i1) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {   // c indexes the SOURCE (BGR) channel; it lands in 2 - c (RGB)
    const float top = __fadd_rn(__fmul_rn(l0w, xform_load(p00 + c)), __fmul_rn(tw.l1, xform_load(p01 + c)));
    const float bot = __fadd_rn(__fmul_rn(l0w, xform_load(p10 + c)), __fmul_rn(tw.l1, xform_load(p11 + c)));
    float v = __fadd_rn(__fmul_rn(l0h, top), __fmul_rn(th.l1, bot));
    if (mode == YB_XFORM_NORMALIZE)
      v = __fdiv_rn(__fsub_rn(v, aff.mean[c]), aff.stdv[c]);
    else if (mode == YB_XFORM_SUBTRACT_MEANS)
      v = __fsub_rn(v, aff.mean[c]);
    else if (mode == YB_XFORM_TO_FLOAT)
      v = __fdiv_rn(v, 255.f);
    rgb[2 - c] = v;
  }
}

// One image of a frame list (yb_infer_frame_list): an [fh][fw][3] uint8 BGR frame resized to the network's H x W.  The
// kernels read a device table of these, one per image, so one launch serves any mix of frame sizes.
struct FrameRef {
  const uint8_t* frame;
  int fh, fw;
  float scale_h, scale_w;   // (float)fh / H, (float)fw / W: ATen's scale, as fast_base_transform computes it
};
inline FrameRef frame_ref(const uint8_t* frame, int fh, int fw, int H, int W) {
  return FrameRef{frame, fh, fw, (float)fh / (float)H, (float)fw / (float)W};
}

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// cudaFuncSetAttribute applies to the CURRENT device: a function-local static of this type remembers, per device,
// whether the attribute of that kernel instantiation has been raised (one process may drive several GPUs).
struct PerDeviceOnce {
  bool done[64] = {};
  bool first() {
    int d = 0;
    cudaGetDevice(&d);
    d &= 63;
    if (done[d]) return false;
    done[d] = true;
    return true;
  }
};

// Launch counter (per handle); every launcher takes one of these.
struct LaunchCounter {
  int64_t n = 0;
};

}  // namespace yb
