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
#include <stdlib.h>
#include <algorithm>
#include "kernels.cuh"

namespace yb {

namespace {

constexpr int MT = 256;  // threads

struct ColTab {  // per output column / row interpolation entry
  int i0, i1;
  float l0, l1;
};

__device__ __forceinline__ ColTab interp_entry(int dst, float scale, int in_size) {
  // ATen area_pixel_compute_source_index, align_corners=False
  float s = fmaxf(__fsub_rn(__fmul_rn(scale, (float)dst + 0.5f), 0.5f), 0.f);
  ColTab t;
  t.i0 = (int)s;
  if (t.i0 > in_size - 1) t.i0 = in_size - 1;
  t.i1 = t.i0 + (t.i0 < in_size - 1 ? 1 : 0);
  t.l1 = __fsub_rn(s, (float)t.i0);
  t.l0 = __fsub_rn(1.f, t.l1);
  return t;
}

// sanitize_coordinates(cast=False) (box_utils.py:327-346)
__device__ __forceinline__ void sanitize(float a, float b, int size, int padding, float* lo, float* hi) {
  float x1 = __fmul_rn(a, (float)size), x2 = __fmul_rn(b, (float)size);
  float mn = fminf(x1, x2), mx = fmaxf(x1, x2);
  *lo = fmaxf(__fsub_rn(mn, (float)padding), 0.f);
  *hi = fminf(__fadd_rn(mx, (float)padding), (float)size);
}

template <int FORMAT>
__global__ void __launch_bounds__(MT)
mask_assembly_kernel(const float* __restrict__ proto, int ph, int pw, int k,
                     const float* __restrict__ coef, const float* __restrict__ box, int n, int out_h,
                     int out_w, int crop, int band, int group, int max_rows, float scale_h,
                     float scale_w, void* __restrict__ masks_v, long long mask_img_stride_bytes) {
  // blockIdx.z = image of the batch (yb_postprocess_batch); every per-image tensor is dense
  proto += (size_t)blockIdx.z * ph * pw * k;
  coef += (size_t)blockIdx.z * n * k;
  box += (size_t)blockIdx.z * n * 4;
  masks_v = reinterpret_cast<unsigned char*>(masks_v) + (size_t)blockIdx.z * mask_img_stride_bytes;
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
      const int head = (int)((4 - (((reinterpret_cast<uintptr_t>(masks_v) / esz) + band_off) & 3)) & 3);
      const int hd = min(head, L);
      const int nq = (L - hd) >> 2;            // aligned 4-element stores
      const int tail = L - hd - 4 * nq;        // < 4 trailing elements
      if (FORMAT == YB_MASK_F32) {
        float* base = reinterpret_cast<float*>(masks_v) + band_off;
        float4* body = reinterpret_cast<float4*>(base + hd);
        for (int q = tid; q < nq; q += MT) __stcs(body + q, make_float4(0.f, 0.f, 0.f, 0.f));
        if (tid < hd) base[tid] = 0.f;
        if (tid < tail) base[hd + 4 * nq + tid] = 0.f;
      } else {
        unsigned char* base = reinterpret_cast<unsigned char*>(masks_v) + band_off;
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
    float cx1 = 0.f, cx2 = (float)pw, cy1 = 0.f, cy2 = (float)ph;
    if (crop) {
      const float* bx = box + (size_t)d * 4;
      sanitize(bx[0], bx[2], pw, 1, &cx1, &cx2);
      sanitize(bx[1], bx[3], ph, 1, &cy1, &cy2);
    }
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
        const float4* pp = reinterpret_cast<const float4*>(proto + ((size_t)pr * pw + c) * k);
        float acc = 0.f;
        for (int j = 0; j < k / 4; ++j) {
          const float4 q = __ldg(pp + j);
          const float4 w4 = __ldg(reinterpret_cast<const float4*>(cf) + j);   // same address in every lane: one L1 broadcast
          acc = fmaf(q.x, w4.x, acc);
          acc = fmaf(q.y, w4.y, acc);
          acc = fmaf(q.z, w4.z, acc);
          acc = fmaf(q.w, w4.w, acc);
        }
        mrows[(size_t)(pr - r_lo) * pw + c] = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-acc)));  // torch.sigmoid
      }
      __syncthreads();
    }

    // ---- stream out the band -------------------------------------------------------------
    if (FORMAT == YB_MASK_BITS) {
      // one warp per output word: lane j evaluates pixel 32*wx + j, the ballot is the packed word
      uint32_t* out = reinterpret_cast<uint32_t*>(masks_v) + (size_t)d * out_h * wpr;
      const int words = (y1 - y0) * wpr;
      if (!any) {
        for (int wi = tid; wi < words; wi += MT) out[(size_t)y0 * wpr + wi] = 0u;   // the band's words are contiguous
      } else {
        // output columns whose interpolation sources can fall inside the crop window (conservative superset,
        // same bounds as the fp32 / uint8 path below): words entirely outside are zero without evaluation
        const int xa = max((int)floorf(__fdiv_rn(cx1 - 0.5f, scale_w) - 0.5f) - 1, 0);
        const int xb = min((int)ceilf(__fdiv_rn(ceilf(cx2) + 0.5f, scale_w) - 0.5f) + 1, out_w);
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
            float top = __fadd_rn(__fmul_rn(ct.l0, ra[ct.i0]), __fmul_rn(ct.l1, ra[ct.i1]));
            float bot = __fadd_rn(__fmul_rn(ct.l0, rb[ct.i0]), __fmul_rn(ct.l1, rb[ct.i1]));
            float v = __fadd_rn(__fmul_rn(rt.l0, top), __fmul_rn(rt.l1, bot));
            bit = v > 0.5f;
          }
          const uint32_t word = __ballot_sync(0xffffffffu, bit);
          if (lane == 0) out[(size_t)y * wpr + wx] = word;
        }
      }
    } else if (any) {
      // ---- phase B: only the output columns whose interpolation sources can fall inside the crop window
      //      (a conservative superset: pixels outside interpolate zeros), only the ones are stored.
      // A pixel x reads source columns i0 = floor(s), i1 = i0 + 1 with s = scale*(x+0.5)-0.5; the columns inside the
      // window are the integers in [ceil(cx1), ceil(cx2)).  i1 >= ceil(cx1) needs s >= ceil(cx1) - 1 (cx1 - 0.5 below is
      // smaller still), i0 < ceil(cx2) needs s < ceil(cx2): x < (ceil(cx2) + 0.5) / scale - 0.5.
      int xa = (int)floorf(__fdiv_rn(cx1 - 0.5f, scale_w) - 0.5f) - 1;
      int xb = (int)ceilf(__fdiv_rn(ceilf(cx2) + 0.5f, scale_w) - 0.5f) + 1;
      xa = max(xa, 0);
      xb = min(xb, out_w);
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
          float top = __fadd_rn(__fmul_rn(ct.l0, ra[ct.i0]), __fmul_rn(ct.l1, ra[ct.i1]));
          float bot = __fadd_rn(__fmul_rn(ct.l0, rb[ct.i0]), __fmul_rn(ct.l1, rb[ct.i1]));
          float v = __fadd_rn(__fmul_rn(rt.l0, top), __fmul_rn(rt.l1, bot));
          if (v > 0.5f) {
            if (FORMAT == YB_MASK_F32)
              reinterpret_cast<float*>(masks_v)[band_off + (size_t)yy * out_w + x] = 1.f;
            else
              reinterpret_cast<unsigned char*>(masks_v)[band_off + (size_t)yy * out_w + x] = 1;
          }
        }
      }
    }
    if (any) __syncthreads();  // mrows reuse
  }
}

// boxes: sanitize_coordinates(cast=False) for x with w, y with h, then .long() (output_utils.py:97-99)
__global__ void boxes_px_kernel(const float* __restrict__ box, int n, int out_h, int out_w,
                                int64_t* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;   // n = total boxes over the batch
  if (i >= n) return;
  float x1, x2, y1, y2;
  sanitize(box[i * 4 + 0], box[i * 4 + 2], out_w, 0, &x1, &x2);
  sanitize(box[i * 4 + 1], box[i * 4 + 3], out_h, 0, &y1, &y2);
  out[i * 4 + 0] = (int64_t)x1;  // truncation toward zero, like Tensor.long()
  out[i * 4 + 1] = (int64_t)y1;
  out[i * 4 + 2] = (int64_t)x2;
  out[i * 4 + 3] = (int64_t)y2;
}

// Cropped sigmoid masks at prototype resolution [n,ph,pw] (FastMaskIoUNet input, output_utils.py:77-82)
__global__ void __launch_bounds__(MT)
proto_masks_kernel(const float* __restrict__ proto, int ph, int pw, int k,
                   const float* __restrict__ coef, const float* __restrict__ box, int crop,
                   float* __restrict__ out) {
  __shared__ float s_coef[128];
  const int r = blockIdx.x, d = blockIdx.y;
  for (int j = threadIdx.x; j < k; j += MT) s_coef[j] = coef[(size_t)d * k + j];
  __syncthreads();
  float cx1 = 0.f, cx2 = (float)pw, cy1 = 0.f, cy2 = (float)ph;
  if (crop) {
    const float* bx = box + (size_t)d * 4;
    sanitize(bx[0], bx[2], pw, 1, &cx1, &cx2);
    sanitize(bx[1], bx[3], ph, 1, &cy1, &cy2);
  }
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
      v = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-acc)));
    }
    out[((size_t)d * ph + r) * pw + c] = v;
  }
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

}  // namespace

void launch_mask_assembly(const float* proto, int ph, int pw, int k, const float* coef,
                          const float* box, int n, int out_h, int out_w, int crop, int mask_format,
                          void* masks, int64_t* boxes_px, float* proto_masks, cudaStream_t stream,
                          LaunchCounter* lc, int batch) {
  if (n <= 0 || batch <= 0) return;
  YB_REQUIRE(batch == 1 || proto_masks == nullptr, "mask_assembly: proto_masks output is per image");
  YB_REQUIRE(k % 4 == 0 && k <= 128, "mask_assembly: mask_dim must be a multiple of 4 and <= 128");
  YB_REQUIRE(out_h > 0 && out_w > 0 && ph > 0 && pw > 0, "mask_assembly: bad sizes");
  const float scale_h = (float)ph / (float)out_h;
  const float scale_w = (float)pw / (float)out_w;
  if (boxes_px) {
    boxes_px_kernel<<<ceil_div(n * batch, 128), 128, 0, stream>>>(box, n * batch, out_h, out_w, boxes_px);
    YB_CHECK_LAUNCH();
    if (lc) lc->n++;
  }
  if (proto_masks) {
    proto_masks_kernel<<<dim3(ph, n), MT, 0, stream>>>(proto, ph, pw, k, coef, box, crop, proto_masks);
    YB_CHECK_LAUNCH();
    if (lc) lc->n++;
  }
  if (masks) {
    YB_REQUIRE((reinterpret_cast<uintptr_t>(masks) & 15) == 0, "mask_assembly: masks must be 16-byte aligned");
    int band = 8;
    int max_rows;
    size_t smem;
    for (;;) {
      max_rows = (int)((double)(band - 1) * scale_h) + 4;
      smem = (size_t)out_w * sizeof(ColTab) + (size_t)max_rows * pw * sizeof(float);
      if (smem <= 200 * 1024 || band == 1) break;
      band = band / 2;
    }
    YB_REQUIRE(smem <= 200 * 1024, "mask_assembly: output too wide for the shared-memory tables");
    const int bands = ceil_div(out_h, band);
    // >= ~4 waves of 8 resident CTAs per SM: enough stores in flight to approach the HBM write rate and a short
    // tail (bands that cross many boxes take several times longer than empty ones); groups stay >= 8 detections
    // so the band's prototype rows are reused from L1.  YB_MASK_CTAS_PER_SM overrides the target (tuning hook).
    static const int ctas_per_sm = getenv("YB_MASK_CTAS_PER_SM") ? std::max(1, atoi(getenv("YB_MASK_CTAS_PER_SM"))) : 32;
    int group = n;
    while (group > 8 && (int64_t)bands * ceil_div(n, group) * batch < (int64_t)ctas_per_sm * 132) group = (group + 1) / 2;
    dim3 grid(bands, ceil_div(n, group), batch);
    const size_t plane = (size_t)out_h * out_w;
    const long long img_stride = (long long)n * (mask_format == YB_MASK_F32 ? plane * 4
                                                : mask_format == YB_MASK_U8 ? plane
                                                                            : (size_t)out_h * ((out_w + 31) / 32) * 4);
#define YB_LAUNCH_MASK(FMT)                                                                       \
  do {                                                                                            \
    if (smem > 48 * 1024)                                                                         \
      YB_CHECK_CUDA(cudaFuncSetAttribute(mask_assembly_kernel<FMT>,                               \
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    mask_assembly_kernel<FMT><<<grid, MT, smem, stream>>>(proto, ph, pw, k, coef, box, n, out_h,  \
                                                         out_w, crop, band, group, max_rows,     \
                                                         scale_h, scale_w, masks, img_stride);   \
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
