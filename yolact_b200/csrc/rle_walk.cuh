// COCO run-length encoding walk shared by mask_rle_kernel (evalops.cu: masks stored in global memory) and
// coco_rle_kernel (cocorle.cu: mask pixels evaluated from the detection, never stored).  Both produce maskApi.c
// rleEncode's runs: column-major order, alternating zero / one runs starting with zeros (counts[0] == 0 when the first
// pixel is set).
//
// The walk is templated on its pixel source.  A source provides
//   void chunk(int c0, int c1)  : called by every thread before the columns [c0, c1) are read (may stage shared memory
//                                 and synchronise the CTA; it also covers column c0 - 1's last row, see first_prev)
//   int operator()(int y, int x): the pixel (0 / 1) of a column in the current chunk, or of column c0 - 1 at row h - 1.
#pragma once
#include "common.cuh"

namespace yb {

// Exclusive block prefix sum of one int per thread (blockDim.x a multiple of 32); *total = the sum over the CTA.
// s_warp holds blockDim.x / 32 ints.
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

// Value changes of one column x of an h-row mask whose ones all lie in rows [ya, yb) and columns [xa, xb) (the rest is
// implied zeros), in ascending column-major position x * h + y.  prev: the pixel before (x, 0) in column-major order.
// The last column of the region also emits the change back to zero at (xb, 0) when its bottom pixel is set.
// EMIT(pos) is called for each change; returns their number.
template <class Src, class Emit>
__device__ __forceinline__ int rle_column(const Src& px, int x, int h, int w, int xb, int ya, int yb, int prev,
                                          Emit&& emit) {
  int cnt = 0;
  const uint32_t col = (uint32_t)x * (uint32_t)h;
  if (ya > 0) {   // rows [0, ya) are zeros
    if (prev) emit(col), ++cnt;
    prev = 0;
  }
  for (int y = ya; y < yb; ++y) {
    const int v = px(y, x);
    if (v != prev) emit(col + (uint32_t)y), ++cnt;
    prev = v;
  }
  if (yb < h) {   // rows [yb, h) are zeros
    if (prev) emit(col + (uint32_t)yb), ++cnt;
    prev = 0;
  }
  if (x == xb - 1 && x + 1 < w && prev) emit(col + (uint32_t)h), ++cnt;   // column xb starts with a zero
  return cnt;
}

// The column-major walk of the region [xa, xb) x [ya, yb) of an h x w mask, NT = blockDim.x columns per chunk, one
// thread per column.  With out == nullptr it only counts; otherwise change j is written to out[j] when j < cap.
// Returns the number of value changes (the same in every thread); runs = changes + 1.
template <class Src>
__device__ int64_t rle_walk(Src& px, int h, int w, int xa, int xb, int ya, int yb, uint32_t* __restrict__ out,
                            int64_t cap, int* s_warp) {
  const int NT = (int)blockDim.x, tid = threadIdx.x;
  int64_t base = 0;   // changes emitted by previous column chunks
  for (int c0 = xa; c0 < xb; c0 += NT) {
    px.chunk(c0, min(c0 + NT, xb));
    const int x = c0 + tid;
    const bool active = x < xb;
    // the pixel before (x, 0): (x - 1, h - 1), a zero unless column x - 1 is in the region and its bottom row too
    const int first_prev = (active && x > xa && yb == h) ? px(h - 1, x - 1) : 0;
    auto none = [](uint32_t) {};
    const int cnt = active ? rle_column(px, x, h, w, xb, ya, yb, first_prev, none) : 0;
    int total;
    const int off = rle_block_scan(cnt, s_warp, &total);
    if (out && active && cnt) {
      int64_t o = base + off;
      rle_column(px, x, h, w, xb, ya, yb, first_prev, [&](uint32_t pos) {
        if (o < cap) out[o] = pos;
        ++o;
      });
    }
    base += total;
  }
  return base;
}

// out[0..T) holds the T change positions of an h*w mask in ascending order: turn them into the T + 1 run lengths
// out[0..T] in place.  Every thread of the CTA calls it.
__device__ __forceinline__ void rle_positions_to_lengths(uint32_t* __restrict__ out, int64_t T, uint32_t hw) {
  const int NT = (int)blockDim.x, tid = threadIdx.x;
  __syncthreads();
  if (tid == 0) out[T] = T ? hw - out[T - 1] : hw;
  __syncthreads();
  // from the back: a chunk only reads entries at or below itself
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

}  // namespace yb
