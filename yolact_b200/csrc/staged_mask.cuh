// One detection row's mask pixels evaluated from shared memory, for the kernels that read a mask straight from the
// detections without writing it (cocorle.cu's run walk, evaliou.cu's IoU words).  The caller sets the fields, calls
// chunk(c0, c1) with every thread before it reads output columns [c0, c1), and then reads pixels with px(y, x).
// Pixels go through mask_math.cuh (lincomb_sigmoid, interp_entry, bilinear4) in the mask kernel's crop-before-upsample
// order, so every pixel is yb_postprocess's, bit for bit.
#pragma once
#include "mask_math.cuh"

namespace yb {

// Pixel source: the cropped sigmoid values of the prototype rows [r_lo, r_lo + nr) and the columns the current chunk
// reads, staged in sig [nr][nc].
struct StagedMask {
  const float* proto;
  const float* cf;   // the row's coefficients
  float* sig;
  int ph, pw, k, xa;
  float cx1, cx2, cy1, cy2, scale_h, scale_w;
  int r_lo, nr, c_lo, nc;
  int staged_a, staged_b;   // output columns whose sources are staged (a chunk already staged is not staged again)

  __device__ void chunk(int c0, int c1) {
    const int a = max(c0 - 1, xa);   // column c0 - 1's last row is the first pixel's predecessor
    if (a == staged_a && c1 == staged_b) return;   // uniform
    staged_a = a, staged_b = c1;
    c_lo = interp_entry(a, scale_w, pw).i0;
    nc = interp_entry(c1 - 1, scale_w, pw).i1 - c_lo + 1;
    __syncthreads();   // the previous chunk's values are no longer read
    for (int idx = threadIdx.x; idx < nr * nc; idx += blockDim.x) {
      const int rr = idx / nc, r = r_lo + rr, c = c_lo + (idx - rr * nc);
      float v = 0.f;
      if ((float)c >= cx1 && (float)c < cx2 && (float)r >= cy1 && (float)r < cy2)
        v = lincomb_sigmoid(proto + ((size_t)r * pw + c) * k, cf, k);
      sig[idx] = v;
    }
    __syncthreads();
  }

  __device__ __forceinline__ int operator()(int y, int x) const {
    const ColTab rt = interp_entry(y, scale_h, ph), ct = interp_entry(x, scale_w, pw);
    return bilinear4(rt, ct, sig + (size_t)(rt.i0 - r_lo) * nc, sig + (size_t)(rt.i1 - r_lo) * nc, ct.i0 - c_lo,
                     ct.i1 - c_lo) > 0.5f;
  }

  // Row d of image `it` at out_h x out_w: the crop window, the output pixels [xa, xb) x [ya, yb) that can be set
  // (window_out_bounds; all four 0 for an empty or NaN window) and the prototype rows those rows read.  No chunk is
  // staged yet.
  __device__ void init(const float* proto_, const float* coef, const float* box, int d, int crop, int ph_, int pw_,
                       int k_, int h, int w, float* sig_, int* pxa, int* pxb, int* pya, int* pyb) {
    proto = proto_;
    cf = coef + (size_t)d * k_;
    sig = sig_;
    ph = ph_, pw = pw_, k = k_;
    scale_h = __fdiv_rn((float)ph, (float)h);
    scale_w = __fdiv_rn((float)pw, (float)w);
    crop_window(box, d, crop, ph, pw, cx1, cx2, cy1, cy2);
    int a, b, c, e;
    window_out_bounds(cx1, cx2, scale_w, w, &a, &b);
    window_out_bounds(cy1, cy2, scale_h, h, &c, &e);
    if (a >= b || c >= e) a = b = c = e = 0;
    xa = a;
    staged_a = staged_b = -1;
    c_lo = nc = 0;
    r_lo = c < e ? interp_entry(c, scale_h, ph).i0 : 0;
    nr = c < e ? interp_entry(e - 1, scale_h, ph).i1 - r_lo + 1 : 0;
    *pxa = a, *pxb = b, *pya = c, *pyb = e;
  }
};

// Columns of prototype a chunk of `span` output columns (and its predecessor) can read at scale_w, as the launchers
// size the staging buffer: ph rows times this many floats.
inline int64_t staged_cols(int span, int pw, int out_w) {
  const float scale_w = (float)pw / (float)out_w;
  const int64_t cols = (int64_t)((double)span * scale_w) + 4;
  return cols < pw ? cols : pw;
}

}  // namespace yb
