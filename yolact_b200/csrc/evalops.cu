// Producers / consumers on either side of the hot path (SURVEY.md section 8f rows 1-2): all HBM-bound
// byte / bit kernels, one launch each.
//
//   fast_base_transform : FastBaseTransform.forward (utils/augmentations.py:616-658): BGR HWC frame
//                         (uint8 or float) -> bilinear resize (F.interpolate, align_corners=False) ->
//                         (x - mean) / std | x - mean | x / 255 -> RGB, NCHW fp32 (the net's input).
//   pack_mask_bits      : float / uint8 0-1 masks -> 1 bit per pixel (YB_MASK_BITS layout).
//   mask_iou_bits       : mask_iou (layers/box_utils.py:98-113) as AND + popcount on packed masks;
//                         eval.py:435-440 (_mask_iou) is the consumer.  Counts are integers, the final
//                         division is the reference's, so the result is bit-identical.
//   box_iou             : jaccard (layers/box_utils.py:54-79), eval.py:442-445 (_bbox_iou).
//   mask_rle            : COCO run-length encoding (column-major runs, starting with zeros) of each mask;
//                         replaces pycocotools.mask.encode in Detections.add_mask (eval.py:320-330).
//   display_blend       : the mask alpha-blend of prep_display (eval.py:186-209) + (img*255).byte().
#include "kernels.cuh"
#include "mask_math.cuh"

namespace yb {

namespace {

// -------------------------------------------------------------------------------------------------
// FastBaseTransform
// -------------------------------------------------------------------------------------------------
// the per-pixel arithmetic is common.cuh xform_pixel, shared with the frame-list stem (stem_tc.cu)
template <typename TIn>
__global__ void __launch_bounds__(256)
fast_base_transform_kernel(const TIn* __restrict__ img, int H, int W, int oh, int ow, float scale_h,
                           float scale_w, int mode, XformAffine aff, float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y, b = blockIdx.z;
  if (x >= ow) return;
  float rgb[3];
  xform_pixel(img + (size_t)b * H * W * 3, W, xform_tap(y, oh, H, scale_h), xform_tap(x, ow, W, scale_w), mode, aff,
              rgb);
  const size_t plane = (size_t)oh * ow;
  float* o = out + (size_t)b * 3 * plane + (size_t)y * ow + x;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[(size_t)c * plane] = rgb[c];
}

// the same from a frame list (yb_infer_frame_list in YB_PREC_F32): image b's frame, size and scales are frames[b]
__global__ void __launch_bounds__(256)
fast_base_transform_list_kernel(const FrameRef* __restrict__ frames, int oh, int ow, int mode, XformAffine aff,
                                float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y, b = blockIdx.z;
  if (x >= ow) return;
  const FrameRef f = frames[b];
  float rgb[3];
  xform_pixel(f.frame, f.fw, xform_tap(y, oh, f.fh, f.scale_h), xform_tap(x, ow, f.fw, f.scale_w), mode, aff, rgb);
  const size_t plane = (size_t)oh * ow;
  float* o = out + (size_t)b * 3 * plane + (size_t)y * ow + x;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[(size_t)c * plane] = rgb[c];
}

// -------------------------------------------------------------------------------------------------
// bit packing + mask IoU
// -------------------------------------------------------------------------------------------------
template <typename TIn>
__global__ void __launch_bounds__(256)
pack_mask_bits_kernel(const TIn* __restrict__ in, int64_t rows, int w, int wpr, uint32_t* __restrict__ out) {
  const int64_t total = rows * wpr;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / wpr;
    const int wx = (int)(i - r * wpr);
    const TIn* src = in + r * w + (int64_t)wx * 32;
    const int xe = min(w - wx * 32, 32);
    uint32_t bits = 0u;
    for (int j = 0; j < xe; ++j) bits |= ((float)src[j] > 0.5f ? 1u : 0u) << j;
    out[i] = bits;
  }
}

constexpr int IOU_THREADS = 128;
// one CTA per (a, b) pair: intersection and both areas by popcount
__global__ void __launch_bounds__(IOU_THREADS)
mask_iou_bits_kernel(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, int64_t words, int m,
                     int iscrowd, float* __restrict__ out) {
  const int i = blockIdx.y, j = blockIdx.x;
  const uint32_t* pa = a + (int64_t)i * words;
  const uint32_t* pb = b + (int64_t)j * words;
  unsigned inter = 0, aa = 0, ab = 0;
  for (int64_t k = threadIdx.x; k < words; k += IOU_THREADS) {
    const uint32_t x = __ldg(pa + k), y = __ldg(pb + k);
    inter += __popc(x & y);
    aa += __popc(x);
    ab += __popc(y);
  }
  __shared__ unsigned red[3][IOU_THREADS / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    inter += __shfl_xor_sync(0xffffffffu, inter, o);
    aa += __shfl_xor_sync(0xffffffffu, aa, o);
    ab += __shfl_xor_sync(0xffffffffu, ab, o);
  }
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = inter;
    red[1][threadIdx.x >> 5] = aa;
    red[2][threadIdx.x >> 5] = ab;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned ti = 0, ta = 0, tb = 0;
    for (int w = 0; w < IOU_THREADS / 32; ++w) {
      ti += red[0][w];
      ta += red[1][w];
      tb += red[2][w];
    }
    // box_utils.py:113 in fp32: intersection / (area_a + area_b - intersection)   |   / area_a
    const float fi = (float)ti, fa = (float)ta, fb = (float)tb;
    out[(int64_t)i * m + j] = iscrowd ? __fdiv_rn(fi, fa) : __fdiv_rn(fi, __fsub_rn(__fadd_rn(fa, fb), fi));
  }
}

__global__ void __launch_bounds__(256)
box_iou_kernel(const float* __restrict__ a, int n, const float* __restrict__ b, int m, int iscrowd,
               float* __restrict__ out) {
  const int64_t total = (int64_t)n * m;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(t / m), j = (int)(t - (int64_t)i * m);
    const float4 A = reinterpret_cast<const float4*>(a)[i];
    const float4 Bx = reinterpret_cast<const float4*>(b)[j];
    // box_utils.py:46-51 (intersect) and :72-79 (jaccard)
    const float iw = fmaxf(__fsub_rn(fminf(A.z, Bx.z), fmaxf(A.x, Bx.x)), 0.f);
    const float ih = fmaxf(__fsub_rn(fminf(A.w, Bx.w), fmaxf(A.y, Bx.y)), 0.f);
    const float inter = __fmul_rn(iw, ih);
    const float area_a = __fmul_rn(__fsub_rn(A.z, A.x), __fsub_rn(A.w, A.y));
    const float area_b = __fmul_rn(__fsub_rn(Bx.z, Bx.x), __fsub_rn(Bx.w, Bx.y));
    const float uni = __fsub_rn(__fadd_rn(area_a, area_b), inter);
    out[t] = iscrowd ? __fdiv_rn(inter, area_a) : __fdiv_rn(inter, uni);
  }
}

// -------------------------------------------------------------------------------------------------
// COCO RLE
// -------------------------------------------------------------------------------------------------
constexpr int RLE_MAX_THREADS = 1024;   // one thread per mask column when w <= 1024 (one pass over the mask)

template <int FORMAT>
struct MaskReader {
  const void* base;
  int w, wpr;
  __device__ __forceinline__ int operator()(int y, int x) const {
    if (FORMAT == YB_MASK_BITS)
      return (int)((reinterpret_cast<const uint32_t*>(base)[(size_t)y * wpr + (x >> 5)] >> (x & 31)) & 1u);
    if (FORMAT == YB_MASK_U8) return reinterpret_cast<const uint8_t*>(base)[(size_t)y * w + x] != 0;
    return reinterpret_cast<const float*>(base)[(size_t)y * w + x] != 0.f;
  }
};

__device__ __forceinline__ int rle_block_scan(int v, int* s_warp, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int n = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += n;
  }
  __syncthreads();
  if (lane == 31) s_warp[wid] = inc;
  __syncthreads();
  int woff = 0, tot = 0;
  const int nwarps = (int)(blockDim.x >> 5);
  for (int w = 0; w < nwarps; ++w) {
    int c = s_warp[w];
    if (w < wid) woff += c;
    tot += c;
  }
  *total = tot;
  return woff + inc - v;
}

// One CTA per mask, one thread per column (up to 1024 per pass).  Thread t walks column c0+t top to bottom (reads are coalesced across the CTA),
// once to count value changes and once to emit their column-major positions; a final in-place pass
// turns positions into run lengths.  counts[0] is the number of leading zeros (0 when the mask starts
// with a one), exactly maskApi.c's rleEncode.
template <int FORMAT>
__global__ void __launch_bounds__(RLE_MAX_THREADS)
mask_rle_kernel(const void* __restrict__ masks, size_t mask_stride_bytes, int h, int w, int wpr,
                uint32_t* __restrict__ counts, int64_t cap, int32_t* __restrict__ nruns) {
  __shared__ int s_warp[RLE_MAX_THREADS / 32];
  const int NT = (int)blockDim.x;
  const int d = blockIdx.x, tid = threadIdx.x;
  MaskReader<FORMAT> px{reinterpret_cast<const uint8_t*>(masks) + (size_t)d * mask_stride_bytes, w, wpr};
  uint32_t* out = counts + (int64_t)d * cap;
  int64_t base = 0;   // transitions emitted by previous column chunks
  for (int c0 = 0; c0 < w; c0 += NT) {
    const int x = c0 + tid;
    const bool active = x < w;
    const int first_prev = (active && x > 0) ? px(h - 1, x - 1) : 0;
    int cnt = 0;
    if (active) {
      int prev = first_prev;
      for (int y = 0; y < h; ++y) {
        const int v = px(y, x);
        cnt += (v != prev);
        prev = v;
      }
    }
    int total;
    int off = rle_block_scan(cnt, s_warp, &total);
    if (active && cnt) {
      int prev = first_prev;
      int64_t o = base + off;
      for (int y = 0; y < h; ++y) {
        const int v = px(y, x);
        if (v != prev) {
          if (o < cap) out[o] = (uint32_t)x * (uint32_t)h + (uint32_t)y;
          ++o;
        }
        prev = v;
      }
    }
    base += total;
  }
  __syncthreads();
  const int64_t T = base;   // number of value changes; runs = T + 1
  if (T + 1 > cap) {
    if (tid == 0) nruns[d] = -(int32_t)(T + 1 < 0x7fffffffll ? T + 1 : 0x7fffffffll);   // overflow: caller must grow cap
    return;
  }
  const uint32_t hw = (uint32_t)h * (uint32_t)w;
  if (tid == 0) {
    out[T] = T ? hw - out[T - 1] : hw;
    nruns[d] = (int32_t)(T + 1);
  }
  __syncthreads();
  // positions -> lengths, in place, from the back (a chunk only reads entries at or below itself)
  for (int64_t hi = T; hi > 0; hi -= NT) {
    const int64_t i = hi - 1 - tid;
    uint32_t cur = 0, prv = 0;
    if (i >= 0) {
      cur = out[i];
      prv = i > 0 ? out[i - 1] : 0u;
    }
    __syncthreads();
    if (i >= 0) out[i] = cur - prv;
    __syncthreads();
  }
}

// -------------------------------------------------------------------------------------------------
// prep_display mask blend
// -------------------------------------------------------------------------------------------------
// img [h,w,3] float; v = img * img_scale (1/255 when the frame is 0..255: eval.py:144 `img / 255.0`).
//   for j: v = v * (1 - alpha*m_j) + m_j*color_j*alpha      (eval.py:197-199, evaluated the way :186-209
//   does: product of the inverse alphas and a cumulative-product weighted sum of the colours)
// out = (v * 255).byte()
template <int FORMAT>
__global__ void __launch_bounds__(256)
display_blend_kernel(const float* __restrict__ img, int img_is_255, const void* __restrict__ masks, int n, int h, int w,
                     int wpr, const float* __restrict__ colors, float alpha, uint8_t* __restrict__ out) {
  extern __shared__ float s_col[];   // [n][3] colour * alpha
  for (int i = threadIdx.x; i < n * 3; i += blockDim.x) s_col[i] = __fmul_rn(colors[i], alpha);
  __syncthreads();
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  const size_t plane_bytes = FORMAT == YB_MASK_BITS ? (size_t)h * wpr * 4 : (FORMAT == YB_MASK_U8 ? (size_t)h * w : (size_t)h * w * 4);
  float prod = 1.f;
  float first[3] = {0.f, 0.f, 0.f}, rest[3] = {0.f, 0.f, 0.f};   // masks_color[0]  |  masks_color_cumul.sum(0)
  const float inv = __fadd_rn(-alpha, 1.f);   // m * (-alpha) + 1 for m == 1
  for (int j = 0; j < n; ++j) {
    MaskReader<FORMAT> px{reinterpret_cast<const uint8_t*>(masks) + (size_t)j * plane_bytes, w, wpr};
    if (px(y, x)) blend_step(j, s_col, inv, prod, first, rest);
  }
  float sum[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) sum[c] = __fadd_rn(first[c], rest[c]);
  const float* p = img + ((size_t)y * w + x) * 3;
  uint8_t* o = out + ((size_t)y * w + x) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    o[c] = blend_out(img_is_255 ? __fdiv_rn(p[c], 255.f) : p[c], prod, sum[c]);
  }
}

inline int grid_for(int64_t total, int block) {
  int64_t g = (total + block - 1) / block;
  const int64_t cap = 132 * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

void launch_fast_base_transform(const void* img, int img_is_u8, int B, int H, int W, int out_h, int out_w, int mode,
                                const float* mean_bgr, const float* std_bgr, float* out, cudaStream_t stream,
                                LaunchCounter* lc) {
  YB_REQUIRE(B > 0 && H > 0 && W > 0 && out_h > 0 && out_w > 0, "fast_base_transform: empty input");
  YB_REQUIRE(out_h <= 65535 && B <= 65535, "fast_base_transform: grid limit");
  XformAffine aff;
  for (int c = 0; c < 3; ++c) {
    aff.mean[c] = mean_bgr[c];
    aff.stdv[c] = std_bgr[c];
  }
  // ATen: scale = (float)in / out when the output size is given (area_pixel_compute_scale)
  const float sh = (float)H / (float)out_h, sw = (float)W / (float)out_w;
  dim3 grid(ceil_div(out_w, 256), out_h, B);
  if (img_is_u8)
    fast_base_transform_kernel<uint8_t><<<grid, 256, 0, stream>>>((const uint8_t*)img, H, W, out_h, out_w, sh, sw, mode,
                                                                  aff, out);
  else
    fast_base_transform_kernel<float><<<grid, 256, 0, stream>>>((const float*)img, H, W, out_h, out_w, sh, sw, mode, aff,
                                                                out);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

void launch_fast_base_transform_list(const FrameRef* d_table, int B, int out_h, int out_w, int mode,
                                     const float* mean_bgr, const float* std_bgr, float* out, cudaStream_t stream,
                                     LaunchCounter* lc) {
  YB_REQUIRE(d_table && B > 0 && out_h > 0 && out_w > 0, "fast_base_transform: empty input");
  YB_REQUIRE(out_h <= 65535 && B <= 65535, "fast_base_transform: grid limit");
  XformAffine aff;
  for (int c = 0; c < 3; ++c) {
    aff.mean[c] = mean_bgr[c];
    aff.stdv[c] = std_bgr[c];
  }
  dim3 grid(ceil_div(out_w, 256), out_h, B);
  fast_base_transform_list_kernel<<<grid, 256, 0, stream>>>(d_table, out_h, out_w, mode, aff, out);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

void launch_pack_mask_bits(const void* in, int in_format, int64_t rows, int w, uint32_t* out, cudaStream_t stream,
                           LaunchCounter* lc) {
  YB_REQUIRE(in_format == YB_MASK_F32 || in_format == YB_MASK_U8, "pack_mask_bits: input must be f32 or u8");
  if (rows == 0) return;
  const int wpr = ceil_div(w, 32);
  const int g = grid_for(rows * wpr, 256);
  if (in_format == YB_MASK_F32)
    pack_mask_bits_kernel<float><<<g, 256, 0, stream>>>((const float*)in, rows, w, wpr, out);
  else
    pack_mask_bits_kernel<uint8_t><<<g, 256, 0, stream>>>((const uint8_t*)in, rows, w, wpr, out);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

void launch_mask_iou_bits(const uint32_t* a, int n, const uint32_t* b, int m, int64_t words, int iscrowd, float* out,
                          cudaStream_t stream, LaunchCounter* lc) {
  if (n == 0 || m == 0) return;
  YB_REQUIRE(n <= 65535, "mask_iou: too many masks");
  dim3 grid(m, n);
  mask_iou_bits_kernel<<<grid, IOU_THREADS, 0, stream>>>(a, b, words, m, iscrowd, out);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

void launch_box_iou(const float* a, int n, const float* b, int m, int iscrowd, float* out, cudaStream_t stream,
                    LaunchCounter* lc) {
  if (n == 0 || m == 0) return;
  box_iou_kernel<<<grid_for((int64_t)n * m, 256), 256, 0, stream>>>(a, n, b, m, iscrowd, out);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

void launch_mask_rle(const void* masks, int mask_format, int n, int h, int w, uint32_t* counts, int64_t cap,
                     int32_t* nruns, cudaStream_t stream, LaunchCounter* lc) {
  if (n == 0) return;
  YB_REQUIRE(h > 0 && w > 0 && (int64_t)h * w < (1ll << 32), "mask_rle: bad mask size");
  YB_REQUIRE(cap >= 1, "mask_rle: cap must be >= 1");
  const int wpr = ceil_div(w, 32);
  const int threads = std::min(RLE_MAX_THREADS, ceil_div(w, 32) * 32);
  switch (mask_format) {
    case YB_MASK_BITS:
      mask_rle_kernel<YB_MASK_BITS><<<n, threads, 0, stream>>>(masks, (size_t)h * wpr * 4, h, w, wpr, counts, cap, nruns);
      break;
    case YB_MASK_U8:
      mask_rle_kernel<YB_MASK_U8><<<n, threads, 0, stream>>>(masks, (size_t)h * w, h, w, wpr, counts, cap, nruns);
      break;
    case YB_MASK_F32:
      mask_rle_kernel<YB_MASK_F32><<<n, threads, 0, stream>>>(masks, (size_t)h * w * 4, h, w, wpr, counts, cap, nruns);
      break;
    default: YB_REQUIRE(false, "mask_rle: unknown mask format");
  }
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

// ---- detection records for the multi-GPU gather (yolact_b200/parallel.py) ---------------------------------------------
// rec[b] = [count, cls[M], score[M], box[M*4], coef[M*k]] as fp32 (class ids < 2^24 and counts are exact in fp32):
// one fixed-size row per image, so that the only data-path collective of a global batch is ONE all_gather.
__global__ void __launch_bounds__(256)
pack_detections_kernel(const float* __restrict__ box, const float* __restrict__ coef, const int64_t* __restrict__ cls,
                       const float* __restrict__ score, const int32_t* __restrict__ count, int M, int k,
                       float* __restrict__ rec) {
  const int b = blockIdx.x;
  const int L = 1 + M * (6 + k);
  float* r = rec + (int64_t)b * L;
  const float* bb = box + (int64_t)b * M * 4;
  const float* cc = coef + (int64_t)b * M * k;
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    float v;
    if (i == 0) v = (float)count[b];
    else if (i < 1 + M) v = (float)cls[(int64_t)b * M + (i - 1)];
    else if (i < 1 + 2 * M) v = score[(int64_t)b * M + (i - 1 - M)];
    else if (i < 1 + 6 * M) v = bb[i - 1 - 2 * M];
    else v = cc[i - 1 - 6 * M];
    r[i] = v;
  }
}
void launch_pack_detections(const float* box, const float* coef, const int64_t* cls, const float* score,
                            const int32_t* count, int B, int M, int k, float* rec, cudaStream_t stream, LaunchCounter* lc) {
  if (B <= 0) return;
  pack_detections_kernel<<<B, 256, 0, stream>>>(box, coef, cls, score, count, M, k, rec);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

void launch_display_blend(const float* img, int img_is_255, const void* masks, int mask_format, int n, int h, int w,
                          const float* colors, float alpha, uint8_t* out, cudaStream_t stream, LaunchCounter* lc) {
  YB_REQUIRE(h > 0 && w > 0 && h <= 65535, "display_blend: bad image size");
  YB_REQUIRE(n >= 0 && n <= 1024, "display_blend: at most 1024 detections");
  const int wpr = ceil_div(w, 32);
  dim3 grid(ceil_div(w, 256), h);
  const size_t smem = (size_t)(n > 0 ? n : 1) * 3 * sizeof(float);
  switch (mask_format) {
    case YB_MASK_BITS:
      display_blend_kernel<YB_MASK_BITS><<<grid, 256, smem, stream>>>(img, img_is_255, masks, n, h, w, wpr, colors, alpha, out);
      break;
    case YB_MASK_U8:
      display_blend_kernel<YB_MASK_U8><<<grid, 256, smem, stream>>>(img, img_is_255, masks, n, h, w, wpr, colors, alpha, out);
      break;
    case YB_MASK_F32:
      display_blend_kernel<YB_MASK_F32><<<grid, 256, smem, stream>>>(img, img_is_255, masks, n, h, w, wpr, colors, alpha, out);
      break;
    default: YB_REQUIRE(false, "display_blend: unknown mask format");
  }
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

}  // namespace yb
