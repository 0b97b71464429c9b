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
template <typename T>
__device__ __forceinline__ T from_f32(float v);
template <>
__device__ __forceinline__ float from_f32<float>(float v) {
  return v;
}
template <>
__device__ __forceinline__ __half from_f32<__half>(float v) {
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
#define YB_LO_SCALE 2048.f
#define YB_LO_INV 4.8828125e-4f   /* 2^-11 */
__device__ __forceinline__ __half lo_from_f32(float r) { return __float2half_rn(r * YB_LO_SCALE); }
__device__ __forceinline__ float lo_to_f32(__half h) { return __half2float(h) * YB_LO_INV; }
__device__ __forceinline__ __half2 lo2_from_f32(float r0, float r1) {
  return __floats2half2_rn(r0 * YB_LO_SCALE, r1 * YB_LO_SCALE);
}
__device__ __forceinline__ float2 lo2_to_f32(__half2 h) {
  const float2 f = __half22float2(h);
  return make_float2(f.x * YB_LO_INV, f.y * YB_LO_INV);
}
// (hi saturates at +-65504; the residual of a saturated value is dropped)
__device__ __forceinline__ void split_f32(float v, __half& hi, __half& lo) {
  const float c = fminf(fmaxf(v, -65504.f), 65504.f);
  hi = __float2half_rn(c);
  lo = lo_from_f32(c - __half2float(hi));
}

__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act) {
    case ACT_RELU: return fmaxf(v, 0.f);
    case ACT_TANH: return tanhf(v);
    case ACT_LEAKY: return v > 0.f ? v : 0.1f * v;
    default: return v;
  }
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
