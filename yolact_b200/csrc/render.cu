// prep_display's mask overlay straight from the detections (eval.py:147-226 with display_text / display_bboxes off):
// no [n,h,w] masks are written.
//
//   render_select_kernel : one CTA per image.  postprocess's score filter (det_score > score_threshold when the threshold
//                          is > 0, output_utils.py:42-50), a stable descending order of the ranking scores (ties to the
//                          lower row), the first top_k rows and the cut at the first score < score_threshold
//                          (eval.py:155-166).  Per drawn slot: palette colour * alpha (eval.py:169-183), crop window and
//                          the output pixels its mask can reach, and the caller's rows (class, score, pixel box).
//   render_kernel        : tiles of TH x TW output pixels of every image of the list (blockIdx.z = image).  Each thread
//                          keeps the blend state of PPT pixels in registers; the CTA streams the drawn detections whose
//                          window meets the tile through shared memory in groups, each holding the cropped sigmoid
//                          values on the prototype rows and columns the tile interpolates from, then blends them in
//                          drawing order.  The frame is read once and the uint8 result written once.
//
// Mask pixels and blend steps go through mask_math.cuh, the functions mask_assembly_kernel and display_blend_kernel use,
// so the image equals postprocess(mask_format='u8') + display_blend on the same rows, bit for bit.
#include <limits.h>
#include <algorithm>
#include "kernels.cuh"
#include "mask_math.cuh"

namespace yb {

namespace {

constexpr int RT = 256;                 // threads
constexpr int TH = 8, TW = 128;         // output tile
constexpr int PPT = TH * TW / RT;       // pixels per thread
constexpr int MIN_SIG = 2 * TH * 2 * TW;  // cropped sigmoid values of one detection on the largest tile

struct RenderSlot {
  int row;                      // detection row
  int xa, xb, ya, yb;           // output pixels its mask can reach (window_out_bounds); empty when nothing is drawn
  float cx1, cx2, cy1, cy2;     // crop window in prototype coordinates
};

struct RenderWork {
  int* counts;        // [B] drawn detections per image
  RenderSlot* slots;  // [B][top_k]
  float* cols;        // [B][top_k][3] palette colour * alpha
};

RenderWork bind_work(void* base, int B, int top_k) {
  char* p = static_cast<char*>(base);
  RenderWork w;
  w.counts = reinterpret_cast<int*>(p);
  p += ((size_t)B * sizeof(int) + 15) / 16 * 16;
  w.slots = reinterpret_cast<RenderSlot*>(p);
  p += ((size_t)B * top_k * sizeof(RenderSlot) + 15) / 16 * 16;
  w.cols = reinterpret_cast<float*>(p);
  return w;
}

__device__ __forceinline__ bool candidate(const float* det_score, int i, float thr) {
  return !(thr > 0.f) || det_score[i] > thr;
}

__global__ void __launch_bounds__(RT)
render_select_kernel(const yb_render_item* __restrict__ items, int ph, int pw, int crop, int top_k, float thr,
                     int class_color, float alpha, const float* __restrict__ palette, int P, RenderWork work) {
  const int b = blockIdx.x;
  const yb_render_item& it = items[b];
  const int n = it.n;
  RenderSlot* sl = work.slots + (size_t)b * top_k;
  __shared__ int s_cand, s_cut;
  if (threadIdx.x == 0) {
    s_cand = 0;
    s_cut = INT_MAX;
  }
  __syncthreads();
  // rank of a candidate = candidates ahead of it in the stable descending order
  int cand = 0;
  for (int i = threadIdx.x; i < n; i += RT) {
    if (!candidate(it.det_score, i, thr)) continue;
    ++cand;
    const float si = it.score[i];
    int rank = 0;
    for (int j = 0; j < n; ++j) {
      if (!candidate(it.det_score, j, thr)) continue;
      const float sj = it.score[j];
      rank += (sj > si || (sj == si && j < i)) ? 1 : 0;
    }
    if (rank < top_k) sl[rank].row = i;
  }
  if (cand) atomicAdd(&s_cand, cand);
  __syncthreads();
  const int m0 = min(s_cand, top_k);
  for (int j = threadIdx.x; j < m0; j += RT)
    if (it.score[sl[j].row] < thr) atomicMin(&s_cut, j);
  __syncthreads();
  const int m = min(m0, s_cut);
  const float scale_h = __fdiv_rn((float)ph, (float)it.h), scale_w = __fdiv_rn((float)pw, (float)it.w);
  for (int j = threadIdx.x; j < top_k; j += RT) {
    RenderSlot s{};
    float* col = work.cols + ((size_t)b * top_k + j) * 3;
    int64_t cls = 0, bx[4] = {0, 0, 0, 0};
    float score = 0.f;
    if (j < m) {
      s.row = sl[j].row;
      cls = it.cls[s.row];
      score = it.score[s.row];
      const int pi = (int)(((class_color ? cls : (int64_t)j) * 5) % P);
#pragma unroll
      for (int c = 0; c < 3; ++c) col[c] = __fmul_rn(palette[pi * 3 + c], alpha);
      if (it.proto) {
        crop_window(it.box, s.row, crop, ph, pw, s.cx1, s.cx2, s.cy1, s.cy2);
        window_out_bounds(s.cx1, s.cx2, scale_w, it.w, &s.xa, &s.xb);
        window_out_bounds(s.cy1, s.cy2, scale_h, it.h, &s.ya, &s.yb);
      }
      // box_px (mask.cu): sanitize_coordinates(cast=False) at the frame size, then .long()
      float x1, x2, y1, y2;
      sanitize(it.box[s.row * 4 + 0], it.box[s.row * 4 + 2], it.w, 0, &x1, &x2);
      sanitize(it.box[s.row * 4 + 1], it.box[s.row * 4 + 3], it.h, 0, &y1, &y2);
      bx[0] = (int64_t)x1;
      bx[1] = (int64_t)y1;
      bx[2] = (int64_t)x2;
      bx[3] = (int64_t)y2;
    }
    sl[j] = s;
    if (it.sel_cls) it.sel_cls[j] = cls;
    if (it.sel_score) it.sel_score[j] = score;
    if (it.sel_box)
      for (int c = 0; c < 4; ++c) it.sel_box[j * 4 + c] = bx[c];
  }
  if (threadIdx.x == 0) {
    work.counts[b] = it.proto ? m : 0;   // no prototypes (cfg.eval_mask_branch off): rows are selected, nothing drawn
    if (it.sel_n) *it.sel_n = m;
  }
}

// Source row (or column) entry e of a tile: the contiguous range lo.. when it holds at most twice the tile's rows, else
// the i0 / i1 pair of each output row (downscaled frames, where output rows are far apart in the prototypes).
__device__ __forceinline__ int src_entry(const ColTab* tab, bool contiguous, int lo, int e) {
  return contiguous ? lo + e : ((e & 1) ? tab[e >> 1].i1 : tab[e >> 1].i0);
}

template <typename T>
__global__ void __launch_bounds__(RT)
render_kernel(const yb_render_item* __restrict__ items, RenderWork work, int top_k, int ph, int pw, int k, float alpha,
              int sig_cap) {
  __shared__ yb_render_item it;
  __shared__ float scale_h, scale_w;
  __shared__ int s_m;
  __shared__ ColTab rtab[TH], ctab[TW];
  extern __shared__ float sig[];   // [group][nre][nce]
  const int tid = threadIdx.x, z = blockIdx.z;
  if (tid == 0) {
    it = items[z];
    scale_h = __fdiv_rn((float)ph, (float)it.h);
    scale_w = __fdiv_rn((float)pw, (float)it.w);
    s_m = work.counts[z];
  }
  __syncthreads();
  const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
  if (x0 >= it.w || y0 >= it.h) return;
  const int x1 = min(x0 + TW, it.w), y1 = min(y0 + TH, it.h);
  const int m = s_m;
  const int tx = tid % TW, ty = tid / TW;   // pixel p of this thread: (y0 + ty + p * RT / TW, x0 + tx)
  constexpr int YSTEP = RT / TW;

  float prod[PPT], first[PPT][3], rest[PPT][3];
#pragma unroll
  for (int p = 0; p < PPT; ++p) {
    prod[p] = 1.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) first[p][c] = rest[p][c] = 0.f;
  }

  if (m > 0) {
    if (tid < y1 - y0) rtab[tid] = interp_entry(y0 + tid, scale_h, ph);
    if (tid < x1 - x0) ctab[tid] = interp_entry(x0 + tid, scale_w, pw);
    __syncthreads();
    const int r_lo = rtab[0].i0, c_lo = ctab[0].i0;
    const int r_span = rtab[y1 - y0 - 1].i1 - r_lo + 1, c_span = ctab[x1 - x0 - 1].i1 - c_lo + 1;
    const bool r_cont = r_span <= 2 * TH, c_cont = c_span <= 2 * TW;
    const int nre = r_cont ? r_span : 2 * (y1 - y0);
    const int nce = c_cont ? c_span : 2 * (x1 - x0);
    const int E = nre * nce;      // <= MIN_SIG <= sig_cap
    const int G = sig_cap / E;    // detections per group
    const RenderSlot* slots = work.slots + (size_t)z * top_k;
    const float* cols = work.cols + (size_t)z * top_k * 3;
    const float inv = __fadd_rn(-alpha, 1.f);   // m * (-alpha) + 1 for m == 1
    // the entries this thread's pixels read: rows ra / rb of each pixel, columns ca / cb
    int ra[PPT], rb[PPT];
#pragma unroll
    for (int p = 0; p < PPT; ++p) {
      const int yy = min(ty + p * YSTEP, y1 - y0 - 1);
      ra[p] = r_cont ? rtab[yy].i0 - r_lo : 2 * yy;
      rb[p] = r_cont ? rtab[yy].i1 - r_lo : 2 * yy + 1;
    }
    const int xx = min(tx, x1 - x0 - 1);
    const int ca = c_cont ? ctab[xx].i0 - c_lo : 2 * xx;
    const int cb = c_cont ? ctab[xx].i1 - c_lo : 2 * xx + 1;
    auto live = [&](const RenderSlot& s) { return s.xa < x1 && s.xb > x0 && s.ya < y1 && s.yb > y0; };

    for (int d0 = 0; d0 < m; d0 += G) {
      const int g1 = min(m, d0 + G);
      __syncthreads();   // the previous group's values are no longer read
      // cropped sigmoid values of the group's detections that reach this tile (zero outside the crop window)
      for (int idx = tid; idx < (g1 - d0) * E; idx += RT) {
        const int g = idx / E, e = idx - g * E;
        const RenderSlot s = slots[d0 + g];
        if (!live(s)) continue;
        const int re = e / nce, ce = e - re * nce;
        const int r = src_entry(rtab, r_cont, r_lo, re), c = src_entry(ctab, c_cont, c_lo, ce);
        float v = 0.f;
        if ((float)c >= s.cx1 && (float)c < s.cx2 && (float)r >= s.cy1 && (float)r < s.cy2)
          v = lincomb_sigmoid(it.proto + ((size_t)r * pw + c) * k, it.coef + (size_t)s.row * k, k);
        sig[idx] = v;
      }
      __syncthreads();
      // blend them in drawing order
      for (int d = d0; d < g1; ++d) {
        const RenderSlot s = slots[d];
        if (!live(s)) continue;   // uniform
        const float* sg = sig + (size_t)(d - d0) * E;
        const ColTab ct = ctab[xx];
#pragma unroll
        for (int p = 0; p < PPT; ++p) {
          const ColTab rt = rtab[min(ty + p * YSTEP, y1 - y0 - 1)];
          if (bilinear4(rt, ct, sg + ra[p] * nce, sg + rb[p] * nce, ca, cb) > 0.5f)
            blend_step(d, cols, inv, prod[p], first[p], rest[p]);
        }
      }
    }
  }

  // out = (frame / 255 * prod + first + rest) * 255, .byte()
  const int x = x0 + tx;
  if (x >= x1) return;
  const T* frame = static_cast<const T*>(it.frame);
#pragma unroll
  for (int p = 0; p < PPT; ++p) {
    const int y = y0 + ty + p * YSTEP;
    if (y >= y1) break;
    const size_t o = ((size_t)y * it.w + x) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c)
      it.out[o + c] = blend_out(__fdiv_rn((float)frame[o + c], 255.f), prod[p], __fadd_rn(first[p][c], rest[p][c]));
  }
}

template <typename T>
size_t render_static_smem() {
  static const size_t bytes = [] {
    cudaFuncAttributes a{};
    YB_CHECK_CUDA(cudaFuncGetAttributes(&a, render_kernel<T>));
    return a.sharedSizeBytes;
  }();
  return bytes;
}

}  // namespace

size_t render_work_bytes(int B, int top_k) {
  return ((size_t)B * sizeof(int) + 15) / 16 * 16 + ((size_t)B * top_k * sizeof(RenderSlot) + 15) / 16 * 16 +
         (size_t)B * top_k * 3 * sizeof(float);
}

void launch_render(const yb_render_item* d_items, const yb_render_item* h_items, int B, int frame_is_u8, int ph, int pw,
                   int k, int crop, int top_k, float score_threshold, int class_color, float alpha,
                   const float* palette, int P, void* work, cudaStream_t stream, LaunchCounter* lc) {
  YB_REQUIRE(B > 0 && B <= 65535 && top_k >= 1 && P >= 1, "render: bad sizes");
  // the grid covers the tallest and widest frame; the group buffer holds at least one detection on any tile, and up to
  // top_k detections on the tiles of the frame that interpolates from the most prototype positions per tile
  int max_h = 0, max_w = 0;
  int64_t per_det = 0;
  for (int b = 0; b < B; ++b) {
    const yb_render_item& it = h_items[b];
    max_h = std::max(max_h, it.h);
    max_w = std::max(max_w, it.w);
    if (it.proto && it.n > 0) {
      YB_REQUIRE(k % 4 == 0 && k <= 128 && ph > 0 && pw > 0, "render: mask_dim must be a multiple of 4 and <= 128");
      const int rows = std::min(2 * TH, (int)((double)(TH - 1) * ph / it.h) + 4);
      const int cols = std::min(2 * TW, (int)((double)(TW - 1) * pw / it.w) + 4);
      per_det = std::max<int64_t>(per_det, (int64_t)rows * cols);
    }
  }
  YB_REQUIRE(ceil_div(max_h, TH) <= 65535, "render: frame too tall");
  const int sig_cap = (int)std::min<int64_t>(std::max<int64_t>(MIN_SIG, per_det * top_k), 6 * MIN_SIG);
  const size_t smem = (size_t)sig_cap * sizeof(float);
  const RenderWork w = bind_work(work, B, top_k);
  render_select_kernel<<<B, RT, 0, stream>>>(d_items, ph, pw, crop, top_k, score_threshold, class_color, alpha, palette,
                                             P, w);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
  const dim3 grid(ceil_div(max_w, TW), ceil_div(max_h, TH), B);
#define YB_LAUNCH_RENDER(T)                                                                                    \
  do {                                                                                                         \
    if (smem + render_static_smem<T>() > 48 * 1024)                                                            \
      YB_CHECK_CUDA(cudaFuncSetAttribute(render_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    render_kernel<T><<<grid, RT, smem, stream>>>(d_items, w, top_k, ph, pw, k, alpha, sig_cap);                \
  } while (0)
  if (frame_is_u8)
    YB_LAUNCH_RENDER(uint8_t);
  else
    YB_LAUNCH_RENDER(float);
#undef YB_LAUNCH_RENDER
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

}  // namespace yb
