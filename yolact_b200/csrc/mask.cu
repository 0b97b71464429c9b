// Mask assembly: ONE kernel for  proto @ coef^T -> sigmoid -> crop -> bilinear upsample -> > 0.5
//
// Reference: postprocess lincomb path (layers/output_utils.py:58-99), crop / sanitize_coordinates
// (layers/box_utils.py:327-373), F.interpolate(..., mode='bilinear', align_corners=False)
// (output_utils.py:91), masks.gt_(0.5) (output_utils.py:94), box sanitise + .long() (:97-99).
//
// The reference materialises [ph,pw,n] (matmul), [ph,pw,n] (sigmoid), 4 boolean crop tensors,
// [n,ph,pw] (permute) and [n,h,w] (interpolate) in HBM.  Here the only HBM traffic is the
// prototype read (L2 resident, 2.4 MB) and the final mask write, which is the roofline:
//     algorithmic bytes = ph*pw*k*4 + n*h*w*sizeof(mask element).
//
// Work decomposition: CTA = (band of BAND output rows, group of detections).  For each detection
// the CTA evaluates the cropped sigmoid mask on the few prototype rows the band interpolates from
// (crop happens BEFORE the upsample, output_utils.py:72-74: each output pixel interpolates four
// already-cropped values), parks them in shared memory and streams out the band.
//
// Every kernel here takes a PostSrc and works on image blockIdx.z (boxes: blockIdx.y): yb_postprocess and
// yb_postprocess_batch pass a strided dense batch, yb_postprocess_list a device table, through the same instances.
#include <stdlib.h>
#include <algorithm>
#include "kernels.cuh"
#include "mask_math.cuh"

namespace yb {

namespace {

constexpr int MT = 256;  // threads

// Image z of a call: the list's table entry, or the dense batch's first image advanced by z strides.
__device__ __forceinline__ yb_post_item post_item(const PostSrc& s, int z) {
  if (s.table) return s.table[z];
  yb_post_item it = s.base;
  it.proto += z * s.proto_step;
  it.coef += z * s.coef_step;
  it.box += z * s.box_step;
  it.masks = static_cast<unsigned char*>(it.masks) + z * s.masks_step_bytes;
  it.boxes_px += z * s.boxes_px_step;
  it.proto_masks += z * s.pm_step;
  return it;
}

// blockIdx.z = image, read through post_item.  The grid and the shared-memory tables are sized for the largest image
// of the call, so CTAs past this image's rows or detections exit at once.  The image's fields stay in shared memory
// and are read where they are used: held in registers through the kernel they would cost 8 more (48 instead of 40).
template <int FORMAT>
__global__ void __launch_bounds__(MT)
mask_assembly_kernel(const PostSrc src, int ph, int pw, int k, int crop, int band, int group, int max_rows) {
  __shared__ yb_post_item it;
  __shared__ float scale_h, scale_w;
  if (threadIdx.x == 0) {
    it = post_item(src, blockIdx.z);
    scale_h = __fdiv_rn((float)ph, (float)it.out_h);
    scale_w = __fdiv_rn((float)pw, (float)it.out_w);
  }
  __syncthreads();
  if (it.masks == nullptr || (int)blockIdx.x * band >= it.out_h || (int)blockIdx.y * group >= it.n) return;
  const float* const& proto = it.proto;
  const float* const& coef = it.coef;
  const float* const& box = it.box;
  // masks are global memory: stores through a pointer read from shared memory would otherwise be generic stores
  const auto masks_v = [] { __builtin_assume(__isGlobal(it.masks)); return it.masks; };
  const int &n = it.n, &out_h = it.out_h, &out_w = it.out_w;
  extern __shared__ unsigned char smem_raw[];
  ColTab* coltab = reinterpret_cast<ColTab*>(smem_raw);                 // [out_w]
  float* mrows = reinterpret_cast<float*>(coltab + out_w);               // [max_rows][pw]

  const int tid = threadIdx.x;
  const int y0 = blockIdx.x * band;
  const int y1 = min(y0 + band, out_h);
  const int d0 = blockIdx.y * group;
  const int d1 = min(d0 + group, n);

  for (int x = tid; x < out_w; x += MT) coltab[x] = interp_entry(x, scale_w, pw);
  // prototype rows this band reads
  const ColTab rt0 = interp_entry(y0, scale_h, ph);
  const ColTab rt1 = interp_entry(y1 - 1, scale_h, ph);
  const int r_lo = rt0.i0;
  const int r_hi = rt1.i1;
  const int nrows = r_hi - r_lo + 1;  // <= max_rows by construction on the host
  __syncthreads();

  const size_t plane = (size_t)out_h * out_w;
  const int wpr = (out_w + 31) >> 5;  // words per row, bit format
  const int L = (y1 - y0) * out_w;    // elements of one detection's band (contiguous in memory)

  // ---- phase A (fp32 / uint8): zero the band of EVERY detection of the group in one flat, memset-like loop of
  //      aligned 4-element stores (streaming: the masks are never read back here).  Phase B below then writes only
  //      the ones, inside the crop window of the detections that reach this band -- a few % of the pixels -- so
  //      the bulk of the output moves at the plain store rate instead of behind per-pixel interpolation code.
  if (FORMAT != YB_MASK_BITS) {
    constexpr size_t esz = (FORMAT == YB_MASK_F32) ? 4 : 1;
    for (int d = d0; d < d1; ++d) {
      const size_t band_off = (size_t)d * plane + (size_t)y0 * out_w;
      // elements up to the next 4-element boundary of the ACTUAL address (the per-image offset of a batched
      // call need not be 16-byte aligned)
      const int head = (int)((4 - (((reinterpret_cast<uintptr_t>(masks_v()) / esz) + band_off) & 3)) & 3);
      const int hd = min(head, L);
      const int nq = (L - hd) >> 2;            // aligned 4-element stores
      const int tail = L - hd - 4 * nq;        // < 4 trailing elements
      if (FORMAT == YB_MASK_F32) {
        float* base = reinterpret_cast<float*>(masks_v()) + band_off;
        float4* body = reinterpret_cast<float4*>(base + hd);
        for (int q = tid; q < nq; q += MT) __stcs(body + q, make_float4(0.f, 0.f, 0.f, 0.f));
        if (tid < hd) base[tid] = 0.f;
        if (tid < tail) base[hd + 4 * nq + tid] = 0.f;
      } else {
        unsigned char* base = reinterpret_cast<unsigned char*>(masks_v()) + band_off;
        uchar4* body = reinterpret_cast<uchar4*>(base + hd);
        for (int q = tid; q < nq; q += MT) body[q] = make_uchar4(0, 0, 0, 0);
        if (tid < hd) base[tid] = 0;
        if (tid < tail) base[hd + 4 * nq + tid] = 0;
      }
    }
    __syncthreads();   // orders the zero stores before this CTA's phase-B stores to the same addresses
  }

  for (int d = d0; d < d1; ++d) {
    // crop window in prototype coordinates (box_utils.py:359-371)
    float cx1, cx2, cy1, cy2;
    crop_window(box, d, crop, ph, pw, cx1, cx2, cy1, cy2);
    // does any prototype row of this band survive the crop?
    bool any = false;
    for (int r = r_lo; r <= r_hi; ++r) any |= ((float)r >= cy1 && (float)r < cy2);
    any &= (cx1 < cx2);

    if (any) {
      // cropped sigmoid(proto . coef) on the prototype rows of this band: zero outside the crop window, and the
      // positions inside it (integer c in [cx1, cx2), r in [cy1, cy2)) enumerated densely so every thread works
      const int c_lo = max((int)ceilf(cx1), 0), c_hi = min((int)ceilf(cx2), pw);
      const int q_lo = max((int)ceilf(cy1), r_lo), q_hi = min((int)ceilf(cy2), r_hi + 1);
      const int cw = c_hi - c_lo;
      for (int pos = tid; pos < nrows * pw; pos += MT) {
        const int r = pos / pw, c = pos - r * pw;
        const int pr = r_lo + r;
        if (!(c >= c_lo && c < c_hi && pr >= q_lo && pr < q_hi)) mrows[pos] = 0.f;
      }
      const float* cf = coef + (size_t)d * k;
      for (int idx = tid; idx < (q_hi - q_lo) * cw; idx += MT) {
        const int rr = idx / cw;
        const int c = c_lo + (idx - rr * cw);
        const int pr = q_lo + rr;
        mrows[(size_t)(pr - r_lo) * pw + c] = lincomb_sigmoid(proto + ((size_t)pr * pw + c) * k, cf, k);
      }
      __syncthreads();
    }

    // ---- stream out the band -------------------------------------------------------------
    if (FORMAT == YB_MASK_BITS) {
      // one warp per output word: lane j evaluates pixel 32*wx + j, the ballot is the packed word
      uint32_t* out = reinterpret_cast<uint32_t*>(masks_v()) + (size_t)d * out_h * wpr;
      const int words = (y1 - y0) * wpr;
      if (!any) {
        for (int wi = tid; wi < words; wi += MT) out[(size_t)y0 * wpr + wi] = 0u;   // the band's words are contiguous
      } else {
        // output columns whose interpolation sources can fall inside the crop window (conservative superset,
        // same bounds as the fp32 / uint8 path below): words entirely outside are zero without evaluation
        int xa, xb;
        window_out_bounds(cx1, cx2, scale_w, out_w, &xa, &xb);
        const int wrp = tid >> 5, lane = tid & 31;
        for (int wi = wrp; wi < words; wi += MT / 32) {
          const int yy = wi / wpr, wx = wi - yy * wpr;
          const int y = y0 + yy;
          const int x = wx * 32 + lane;
          const ColTab rt = interp_entry(y, scale_h, ph);
          // both source rows outside the crop window -> the whole output row is zero
          const bool row_live = ((float)rt.i0 >= cy1 && (float)rt.i0 < cy2) || ((float)rt.i1 >= cy1 && (float)rt.i1 < cy2);
          if (!row_live || wx * 32 + 32 <= xa || wx * 32 >= xb) {   // warp-uniform
            if (lane == 0) out[(size_t)y * wpr + wx] = 0u;
            continue;
          }
          bool bit = false;
          if (x < out_w) {
            const float* ra = mrows + (size_t)(rt.i0 - r_lo) * pw;
            const float* rb = mrows + (size_t)(rt.i1 - r_lo) * pw;
            const ColTab ct = coltab[x];
            bit = bilinear4(rt, ct, ra, rb, ct.i0, ct.i1) > 0.5f;
          }
          const uint32_t word = __ballot_sync(0xffffffffu, bit);
          if (lane == 0) out[(size_t)y * wpr + wx] = word;
        }
      }
    } else if (any) {
      // ---- phase B: only the output columns whose interpolation sources can fall inside the crop window
      //      (window_out_bounds), only the ones are stored.
      int xa, xb;
      window_out_bounds(cx1, cx2, scale_w, out_w, &xa, &xb);
      const size_t band_off = (size_t)d * plane + (size_t)y0 * out_w;
      for (int yy = 0; yy < y1 - y0; ++yy) {
        const ColTab rt = interp_entry(y0 + yy, scale_h, ph);   // uniform
        // both source rows outside the crop window -> the whole output row stays zero
        if (!(((float)rt.i0 >= cy1 && (float)rt.i0 < cy2) || ((float)rt.i1 >= cy1 && (float)rt.i1 < cy2))) continue;
        const float* ra = mrows + (size_t)(rt.i0 - r_lo) * pw;
        const float* rb = mrows + (size_t)(rt.i1 - r_lo) * pw;
        for (int x = xa + tid; x < xb; x += MT) {
          const ColTab ct = coltab[x];
          if (!(((float)ct.i0 >= cx1 && (float)ct.i0 < cx2) || ((float)ct.i1 >= cx1 && (float)ct.i1 < cx2))) continue;
          if (bilinear4(rt, ct, ra, rb, ct.i0, ct.i1) > 0.5f) {
            if (FORMAT == YB_MASK_F32)
              reinterpret_cast<float*>(masks_v())[band_off + (size_t)yy * out_w + x] = 1.f;
            else
              reinterpret_cast<unsigned char*>(masks_v())[band_off + (size_t)yy * out_w + x] = 1;
          }
        }
      }
    }
    if (any) __syncthreads();  // mrows reuse
  }
}

// boxes: sanitize_coordinates(cast=False) for x with w, y with h, then .long() (output_utils.py:97-99)
__device__ __forceinline__ void box_px(const float* __restrict__ box, int i, int out_h, int out_w,
                                       int64_t* __restrict__ out) {
  float x1, x2, y1, y2;
  sanitize(box[i * 4 + 0], box[i * 4 + 2], out_w, 0, &x1, &x2);
  sanitize(box[i * 4 + 1], box[i * 4 + 3], out_h, 0, &y1, &y2);
  out[i * 4 + 0] = (int64_t)x1;  // truncation toward zero, like Tensor.long()
  out[i * 4 + 1] = (int64_t)y1;
  out[i * 4 + 2] = (int64_t)x2;
  out[i * 4 + 3] = (int64_t)y2;
}

__global__ void boxes_px_kernel(const PostSrc src) {
  const yb_post_item it = post_item(src, blockIdx.y);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (it.boxes_px == nullptr || i >= it.n) return;
  box_px(it.box, i, it.out_h, it.out_w, it.boxes_px);
}

// Cropped sigmoid masks at prototype resolution [n,ph,pw] (FastMaskIoUNet input, output_utils.py:77-82): prototype
// row r of detection d
__device__ __forceinline__ void proto_masks_row(const float* __restrict__ proto, int ph, int pw, int k,
                                                const float* __restrict__ coef, const float* __restrict__ box,
                                                int crop, float* __restrict__ out, int r, int d) {
  __shared__ float s_coef[128];
  for (int j = threadIdx.x; j < k; j += MT) s_coef[j] = coef[(size_t)d * k + j];
  __syncthreads();
  float cx1, cx2, cy1, cy2;
  crop_window(box, d, crop, ph, pw, cx1, cx2, cy1, cy2);
  for (int c = threadIdx.x; c < pw; c += MT) {
    float v = 0.f;
    if ((float)c >= cx1 && (float)c < cx2 && (float)r >= cy1 && (float)r < cy2) {
      const float4* pp = reinterpret_cast<const float4*>(proto + ((size_t)r * pw + c) * k);
      float acc = 0.f;
      for (int j = 0; j < k / 4; ++j) {
        float4 q = __ldg(pp + j);
        acc = fmaf(q.x, s_coef[4 * j + 0], acc);
        acc = fmaf(q.y, s_coef[4 * j + 1], acc);
        acc = fmaf(q.z, s_coef[4 * j + 2], acc);
        acc = fmaf(q.w, s_coef[4 * j + 3], acc);
      }
      v = sigmoid_rn(acc);
    }
    out[((size_t)d * ph + r) * pw + c] = v;
  }
}

// blockIdx.z = image.  yb_postprocess_list's callers point consecutive images at consecutive rows of one
// [sum n, ph, pw] buffer, so that maskiou_net runs once on all of them.
__global__ void __launch_bounds__(MT)
proto_masks_kernel(const PostSrc src, int ph, int pw, int k, int crop) {
  const yb_post_item it = post_item(src, blockIdx.z);
  if (it.proto_masks == nullptr || (int)blockIdx.y >= it.n) return;
  proto_masks_row(it.proto, ph, pw, k, it.coef, it.box, crop, it.proto_masks, blockIdx.x, blockIdx.y);
}

// out[i] = max_{h,w} x[i,h,w,cls[i]]   (F.max_pool2d over the full map + gather);
// cls == nullptr: out[i][c] for every channel (grid.y = C), i.e. FastMaskIoUNet.forward itself
__global__ void maxpool_gather_kernel(const float* __restrict__ x, int HW, int C,
                                      const int64_t* __restrict__ cls, float* __restrict__ out) {
  const int i = blockIdx.x;
  const int c = cls ? (int)cls[i] : (int)blockIdx.y;
  float m = -INFINITY;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) m = fmaxf(m, x[((size_t)i * HW + p) * C + c]);
#pragma unroll
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ float s[32];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    float r = s[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) r = fmaxf(r, s[w]);
    if (cls)
      out[i] = r;
    else
      out[(size_t)i * C + c] = r;
  }
}

// Rows per band (the largest of 8, 4, 2, 1 whose tables fit in 200 KB of shared memory), prototype rows per band and
// dynamic shared memory of mask_assembly for an output width out_w and vertical scale scale_h = ph / out_h.
void mask_band(float scale_h, int out_w, int pw, int* band, int* max_rows, size_t* smem) {
  *band = 8;
  for (;;) {
    *max_rows = (int)((double)(*band - 1) * scale_h) + 4;
    *smem = (size_t)out_w * sizeof(ColTab) + (size_t)*max_rows * pw * sizeof(float);
    if (*smem <= 200 * 1024 || *band == 1) break;
    *band = *band / 2;
  }
  YB_REQUIRE(*smem <= 200 * 1024, "mask_assembly: output too wide for the shared-memory tables");
}

// Detections per CTA: >= ~4 waves of 8 resident CTAs per SM, enough stores in flight to approach the HBM write rate
// and a short tail (bands that cross many boxes take several times longer than empty ones); groups stay >= 8
// detections so the band's prototype rows are reused from L1.
int mask_group(int bands, int n, int batch) {
  const int ctas_per_sm = 32;
  int group = n;
  while (group > 8 && (int64_t)bands * ceil_div(n, group) * batch < (int64_t)ctas_per_sm * 132) group = (group + 1) / 2;
  return group;
}

// Static shared memory of a mask_assembly instance.  Without opting in, a kernel may use 48 KB of shared memory in all,
// static and dynamic together.
template <int FORMAT>
size_t mask_static_smem() {
  static const size_t bytes = [] {
    cudaFuncAttributes a{};
    YB_CHECK_CUDA(cudaFuncGetAttributes(&a, mask_assembly_kernel<FORMAT>));
    return a.sharedSizeBytes;
  }();
  return bytes;
}

}  // namespace

PostSrc dense_post_src(const yb_post_item& first, int ph, int pw, int k, int mask_format) {
  PostSrc s{};
  s.base = first;
  const long long n = first.n;
  const long long plane = (long long)first.out_h * first.out_w;
  s.proto_step = (long long)ph * pw * k;
  s.coef_step = n * k;
  s.box_step = n * 4;
  s.masks_step_bytes = n * (mask_format == YB_MASK_F32 ? plane * 4
                            : mask_format == YB_MASK_U8 ? plane
                                                        : (long long)first.out_h * ((first.out_w + 31) / 32) * 4);
  s.boxes_px_step = n * 4;
  s.pm_step = n * ph * pw;
  // a null output stays null in every image, so the kernels' "not wanted" checks hold for the whole batch
  if (!first.masks) s.masks_step_bytes = 0;
  if (!first.boxes_px) s.boxes_px_step = 0;
  if (!first.proto_masks) s.pm_step = 0;
  return s;
}

void launch_mask_assembly(const PostSrc& src, const yb_post_item* h_items, int B, int ph, int pw, int k, int crop,
                          int mask_format, cudaStream_t stream, LaunchCounter* lc) {
  YB_REQUIRE(k % 4 == 0 && k <= 128, "mask_assembly: mask_dim must be a multiple of 4 and <= 128");
  YB_REQUIRE(ph > 0 && pw > 0, "mask_assembly: bad sizes");
  // the grid covers the most rows of any image; the masks' grid and shared-memory tables also the tallest and widest
  // output and the largest vertical scale (the smallest out_h) among the images that want masks
  int max_n = 0, mask_n = 0, max_h = 0, max_w = 0, min_h = 0;
  bool any_boxes = false, any_pm = false;
  for (int b = 0; b < (src.table ? B : 1); ++b) {
    const yb_post_item& it = h_items[b];
    YB_REQUIRE(it.n >= 0 && it.out_h > 0 && it.out_w > 0, "mask_assembly: bad sizes");
    if (it.n == 0) continue;
    max_n = std::max(max_n, it.n);
    any_boxes |= it.boxes_px != nullptr;
    any_pm |= it.proto_masks != nullptr;
    if (it.masks) {
      YB_REQUIRE((reinterpret_cast<uintptr_t>(it.masks) & 15) == 0, "mask_assembly: masks must be 16-byte aligned");
      mask_n = std::max(mask_n, it.n);
      max_h = std::max(max_h, it.out_h);
      max_w = std::max(max_w, it.out_w);
      min_h = min_h ? std::min(min_h, it.out_h) : it.out_h;
    }
  }
  if (any_boxes) {
    boxes_px_kernel<<<dim3(ceil_div(max_n, 128), B), 128, 0, stream>>>(src);
    YB_CHECK_LAUNCH();
    if (lc) lc->n++;
  }
  if (any_pm) {
    proto_masks_kernel<<<dim3(ph, max_n, B), MT, 0, stream>>>(src, ph, pw, k, crop);
    YB_CHECK_LAUNCH();
    if (lc) lc->n++;
  }
  if (mask_n > 0) {
    int band, max_rows;
    size_t smem;
    mask_band((float)ph / (float)min_h, max_w, pw, &band, &max_rows, &smem);
    const int bands = ceil_div(max_h, band);
    const int group = mask_group(bands, mask_n, B);
    const dim3 grid(bands, ceil_div(mask_n, group), B);
#define YB_LAUNCH_MASK(FMT)                                                                                  \
  do {                                                                                                       \
    if (smem + mask_static_smem<FMT>() > 48 * 1024)                                                         \
      YB_CHECK_CUDA(cudaFuncSetAttribute(mask_assembly_kernel<FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                         (int)smem));                                                        \
    mask_assembly_kernel<FMT><<<grid, MT, smem, stream>>>(src, ph, pw, k, crop, band, group, max_rows);      \
  } while (0)
    switch (mask_format) {
      case YB_MASK_F32: YB_LAUNCH_MASK(YB_MASK_F32); break;
      case YB_MASK_U8: YB_LAUNCH_MASK(YB_MASK_U8); break;
      case YB_MASK_BITS: YB_LAUNCH_MASK(YB_MASK_BITS); break;
      default: YB_REQUIRE(false, "mask_assembly: unknown mask format");
    }
#undef YB_LAUNCH_MASK
    YB_CHECK_LAUNCH();
    if (lc) lc->n++;
  }
}

void launch_maxpool_gather(const float* x_nhwc, int n, int H, int W, int C, const int64_t* cls,
                           float* out, cudaStream_t stream, LaunchCounter* lc) {
  if (n <= 0) return;
  maxpool_gather_kernel<<<dim3(n, cls ? 1 : C), 128, 0, stream>>>(x_nhwc, H * W, C, cls, out);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

}  // namespace yb
