// Per-pixel arithmetic shared by the mask kernels (mask.cu), the display blend (evalops.cu) and the fused mask render
// (render.cu).  Every kernel that produces or consumes a mask pixel evaluates it through these functions, so their
// results agree bit for bit by construction.  The box IoU of jaccard is here too, for box_iou_kernel (evalops.cu) and
// eval_iou_kernel (evaliou.cu).
#pragma once
#include "common.cuh"

namespace yb {

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

// sanitize_coordinates(cast=False) (box_utils.py:327-346).  torch.min, torch.max and clamp propagate NaN where
// fminf / fmaxf drop it: a NaN coordinate makes both ends NaN, so every crop comparison fails (an empty mask) and the
// pixel box converts NaN exactly as Tensor.long() does.
__device__ __forceinline__ void sanitize(float a, float b, int size, int padding, float* lo, float* hi) {
  float x1 = __fmul_rn(a, (float)size), x2 = __fmul_rn(b, (float)size);
  float mn = fminf(x1, x2), mx = fmaxf(x1, x2);
  *lo = fmaxf(__fsub_rn(mn, (float)padding), 0.f);
  *hi = fminf(__fadd_rn(mx, (float)padding), (float)size);
  if (isnan(x1) || isnan(x2)) *lo = *hi = __int_as_float(0x7fffffff);
}

// crop window of one detection in prototype coordinates (box_utils.py:359-371); the whole map without crop.  A position
// (r, c) survives the crop when cx1 <= c < cx2 and cy1 <= r < cy2, i.e. c in [ceil(cx1), ceil(cx2)).
__device__ __forceinline__ void crop_window(const float* box, int d, int crop, int ph, int pw, float& cx1, float& cx2,
                                            float& cy1, float& cy2) {
  cx1 = 0.f, cx2 = (float)pw, cy1 = 0.f, cy2 = (float)ph;
  if (crop) {
    const float* bx = box + (size_t)d * 4;
    sanitize(bx[0], bx[2], pw, 1, &cx1, &cx2);
    sanitize(bx[1], bx[3], ph, 1, &cy1, &cy2);
  }
}

// Output columns [xa, xb) whose interpolation sources can fall inside the crop window [cx1, cx2) (a conservative
// superset: pixels outside interpolate zeros).  A pixel x reads source columns i0 = floor(s), i1 = i0 + 1 with
// s = scale*(x+0.5)-0.5; the columns inside the window are the integers in [ceil(cx1), ceil(cx2)).  i1 >= ceil(cx1)
// needs s >= ceil(cx1) - 1 (cx1 - 0.5 below is smaller still), i0 < ceil(cx2) needs s < ceil(cx2):
// x < (ceil(cx2) + 0.5) / scale - 0.5.  Rows are the same with the vertical window and scale.  An empty or NaN window
// (!(c1 < c2)) reaches no pixel.
__device__ __forceinline__ void window_out_bounds(float c1, float c2, float scale, int out_size, int* a, int* b) {
  if (!(c1 < c2)) {
    *a = *b = 0;
    return;
  }
  *a = max((int)floorf(__fdiv_rn(c1 - 0.5f, scale) - 0.5f) - 1, 0);
  *b = min((int)ceilf(__fdiv_rn(ceilf(c2) + 0.5f, scale) - 0.5f) + 1, out_size);
}

// torch.sigmoid of one lincomb value
__device__ __forceinline__ float sigmoid_rn(float acc) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-acc))); }

// sigmoid(proto . coef) at one prototype position: pp = proto + (r * pw + c) * k, cf = coef of the detection (16-byte
// aligned), k % 4 == 0; the products accumulate in k order with one fmaf each
__device__ __forceinline__ float lincomb_sigmoid(const float* pp, const float* cf, int k) {
  const float4* p4 = reinterpret_cast<const float4*>(pp);
  float acc = 0.f;
  // not unrolled: an unrolled body keeps more loads in flight than the 40 registers that leave 6 CTAs per SM
#pragma unroll 1
  for (int j = 0; j < k / 4; ++j) {
    const float4 q = __ldg(p4 + j);
    const float4 w4 = __ldg(reinterpret_cast<const float4*>(cf) + j);   // same address in every lane: one L1 broadcast
    acc = fmaf(q.x, w4.x, acc);
    acc = fmaf(q.y, w4.y, acc);
    acc = fmaf(q.z, w4.z, acc);
    acc = fmaf(q.w, w4.w, acc);
  }
  return sigmoid_rn(acc);
}

// bilinear value of an output pixel from its four cropped sigmoid sources: rows ra (source row rt.i0) and rb (rt.i1),
// each read at columns c0 (source column ct.i0) and c1 (ct.i1); the mask is value > 0.5
__device__ __forceinline__ float bilinear4(const ColTab& rt, const ColTab& ct, const float* ra, const float* rb, int c0,
                                           int c1) {
  float top = __fadd_rn(__fmul_rn(ct.l0, ra[c0]), __fmul_rn(ct.l1, ra[c1]));
  float bot = __fadd_rn(__fmul_rn(ct.l0, rb[c0]), __fmul_rn(ct.l1, rb[c1]));
  return __fadd_rn(__fmul_rn(rt.l0, top), __fmul_rn(rt.l1, bot));
}

// ---- prep_display's blend (eval.py:186-209,226), one pixel ---------------------------------------------------------
// For the masks drawn at this pixel, in drawing order j, with col = colour_j * alpha and inv = 1 - alpha:
//   masks_color[0] (first) | the cumulative-product weighted sum of the others (rest) | the product of the inverse
//   alphas (prod)
// (cols: [.][3] colours * alpha, j's at cols + 3 * j)
__device__ __forceinline__ void blend_step(int j, const float* cols, float inv, float& prod, float (&first)[3],
                                           float (&rest)[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    if (j == 0)
      first[c] = cols[c];
    else
      rest[c] = __fadd_rn(rest[c], __fmul_rn(cols[j * 3 + c], prod));
  }
  prod = __fmul_rn(prod, inv);
}

// (v * prod + first + rest) * 255, .byte() (truncation); v = the frame's value scaled to 0..1.  dim: the value is first
// scaled by the fps box's 0.6 (eval.py:219, `*= 0.6` on an fp32 tensor: torch rounds the scalar to fp32)
__device__ __forceinline__ uint8_t blend_out(float v, float prod, float sum, bool dim = false) {
  v = __fadd_rn(__fmul_rn(v, prod), sum);
  if (dim) v = __fmul_rn(v, 0.6f);
  v = __fmul_rn(v, 255.f);
  return (uint8_t)(int)fminf(fmaxf(v, 0.f), 255.f);
}

// ---- jaccard (box_utils.py:46-51 intersect, :72-79 jaccard) of one pair of x1y1x2y2 boxes ---------------------------
__device__ __forceinline__ float box_jaccard(float4 A, float4 B, int iscrowd) {
  const float iw = fmaxf(__fsub_rn(fminf(A.z, B.z), fmaxf(A.x, B.x)), 0.f);
  const float ih = fmaxf(__fsub_rn(fminf(A.w, B.w), fmaxf(A.y, B.y)), 0.f);
  const float inter = __fmul_rn(iw, ih);
  const float area_a = __fmul_rn(__fsub_rn(A.z, A.x), __fsub_rn(A.w, A.y));
  const float area_b = __fmul_rn(__fsub_rn(B.z, B.x), __fsub_rn(B.w, B.y));
  const float uni = __fsub_rn(__fadd_rn(area_a, area_b), inter);
  return iscrowd ? __fdiv_rn(inter, area_a) : __fdiv_rn(inter, uni);
}

// mask_iou (box_utils.py:113) in fp32 from the popcounts: intersection / (area_a + area_b - intersection), or / area_a
// when iscrowd; 0 / 0 is NaN as in the reference
__device__ __forceinline__ float mask_iou_counts(unsigned inter, unsigned area_a, unsigned area_b, int iscrowd) {
  const float fi = (float)inter, fa = (float)area_a, fb = (float)area_b;
  return iscrowd ? __fdiv_rn(fi, fa) : __fdiv_rn(fi, __fsub_rn(__fadd_rn(fa, fb), fi));
}

}  // namespace yb
