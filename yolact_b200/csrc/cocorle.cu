// eval.py's --output_coco_json masks straight from the detections (Detections.add_mask, eval.py:320-330): for every row
// of every image of a list, the pycocotools rleToString string of the mask yb_postprocess would produce for it
// (crop_masks, bilinear, > 0.5), without writing the mask anywhere.
//
//   coco_rle_kernel : one CTA per detection row (blockIdx.x = row, blockIdx.y = image).  Only the output pixels inside
//                     window_out_bounds of the row's crop window can be set; the run walk of rle_walk.cuh visits those
//                     columns and rows and treats everything else as zeros.  For each chunk of up to blockDim.x output
//                     columns the cropped sigmoid values of the prototype rectangle the chunk interpolates from are
//                     staged once in shared memory; each pixel is then bilinear4 of four staged values, > 0.5.
//                     Pass 1 counts the value changes, the row reserves its runs in the caller's run arena (atomic
//                     add), pass 2 writes the change positions there, the shared positions -> lengths pass turns them
//                     into runs, and the CTA writes rleToString's characters into the caller's character arena
//                     (character lengths in parallel, a block scan for the offsets, an atomic add for the space).
//
// Mask pixels come from staged_mask.cuh's StagedMask, which evaluates them through mask_math.cuh (crop_window,
// lincomb_sigmoid, interp_entry, bilinear4), the functions mask_assembly_kernel uses, with the same crop-before-upsample
// order, so the runs are yb_mask_rle's of yb_postprocess's masks, bit for bit.
#include <algorithm>
#include "kernels.cuh"
#include "rle_walk.cuh"
#include "staged_mask.cuh"

namespace yb {

namespace {

constexpr int CR_MAX_THREADS = 1024;

// maskApi.c rleToString of one count: x = cnts[i] - cnts[i-2] for i > 2, 5 bits per character from the low end, 0x20
// while more follow, + 48.  At most 7 characters for a 32-bit count.
__device__ __forceinline__ int64_t rle_delta(const uint32_t* cnts, int64_t i) {
  return (int64_t)cnts[i] - (i > 2 ? (int64_t)cnts[i - 2] : 0);
}
__device__ __forceinline__ int rle_chars(int64_t x, char* dst) {
  int n = 0;
  for (bool more = true; more; ++n) {
    int c = (int)(x & 0x1f);
    x >>= 5;
    more = (c & 0x10) ? x != -1 : x != 0;
    if (more) c |= 0x20;
    if (dst) dst[n] = (char)(c + 48);
  }
  return n;
}

struct CocoOut {
  uint32_t* runs;              // run arena
  int64_t runs_cap;
  char* chars;                 // character arena
  int64_t chars_cap;
  int64_t* row_off;            // [rows]
  int32_t* row_len;            // [rows]
  unsigned long long* need;    // [2]: runs and characters reserved by all rows
};

__global__ void __launch_bounds__(CR_MAX_THREADS)
coco_rle_kernel(const yb_post_item* __restrict__ items, int ph, int pw, int k, int crop, CocoOut o) {
  __shared__ int s_warp[CR_MAX_THREADS / 32];
  __shared__ yb_post_item it;
  __shared__ long long s_runs, s_chars;
  extern __shared__ float sig[];
  const int b = blockIdx.y, d = blockIdx.x, tid = threadIdx.x, NT = blockDim.x;
  if (tid == 0) it = items[b];
  __syncthreads();
  if (d >= it.n) return;   // uniform
  // the global row: rows of the images before this one, then d
  int pre = 0;
  for (int j = tid; j < b; j += NT) pre += items[j].n;
  int before;
  rle_block_scan(pre, s_warp, &before);
  const int64_t row = (int64_t)before + d;
  const int h = it.out_h, w = it.out_w;

  StagedMask px;
  int xa, xb, ya, yb;   // the output pixels that can be set
  px.init(it.proto, it.coef, it.box, d, crop, ph, pw, k, h, w, sig, &xa, &xb, &ya, &yb);

  // pass 1: the number of value changes T; the mask has T + 1 runs
  const int64_t T = rle_walk(px, h, w, xa, xb, ya, yb, nullptr, 0, s_warp);
  if (tid == 0) {
    const long long off = (long long)atomicAdd(o.need, (unsigned long long)(T + 1));
    s_runs = off + T + 1 <= o.runs_cap ? off : -1;
    // a row without room for its runs cannot count its characters: it reserves the 7-per-run bound instead, so that
    // one retry with the reported sizes has room for every row
    if (s_runs < 0) {
      atomicAdd(o.need + 1, (unsigned long long)(7 * (T + 1)));
      o.row_off[row] = 0;
      o.row_len[row] = -1;
    }
  }
  __syncthreads();
  if (s_runs < 0) return;   // uniform
  uint32_t* runs = o.runs + s_runs;
  // pass 2: the change positions (a single chunk is still staged from pass 1), then the run lengths
  rle_walk(px, h, w, xa, xb, ya, yb, runs, T + 1, s_warp);
  rle_positions_to_lengths(runs, T, (uint32_t)h * (uint32_t)w);

  // rleToString: characters per count, then the row's space, then the characters at their scanned offsets
  int64_t nch = 0;
  for (int64_t i0 = 0; i0 <= T; i0 += NT) {
    const int64_t i = i0 + tid;
    int t;
    rle_block_scan(i <= T ? rle_chars(rle_delta(runs, i), nullptr) : 0, s_warp, &t);
    nch += t;
  }
  if (tid == 0) {
    const long long off = (long long)atomicAdd(o.need + 1, (unsigned long long)nch);
    const bool fits = off + nch <= o.chars_cap;
    s_chars = fits ? off : -1;
    o.row_off[row] = fits ? off : 0;
    o.row_len[row] = fits ? (int32_t)nch : -1;
  }
  __syncthreads();
  if (s_chars < 0) return;   // uniform
  char* dst = o.chars + s_chars;
  int64_t base = 0;
  for (int64_t i0 = 0; i0 <= T; i0 += NT) {
    const int64_t i = i0 + tid;
    const int64_t x = i <= T ? rle_delta(runs, i) : 0;
    int t;
    const int at = rle_block_scan(i <= T ? rle_chars(x, nullptr) : 0, s_warp, &t);
    if (i <= T) rle_chars(x, dst + base + at);
    base += t;
  }
}

size_t coco_rle_static_smem() {
  static const size_t bytes = [] {
    cudaFuncAttributes a{};
    YB_CHECK_CUDA(cudaFuncGetAttributes(&a, coco_rle_kernel));
    return a.sharedSizeBytes;
  }();
  return bytes;
}

}  // namespace

void launch_coco_rle(const yb_post_item* d_items, const yb_post_item* h_items, int B, int ph, int pw, int k, int crop,
                     uint32_t* runs, int64_t runs_cap, char* chars, int64_t chars_cap, int64_t* row_off,
                     int32_t* row_len, int64_t* need, cudaStream_t stream, LaunchCounter* lc) {
  YB_REQUIRE(B >= 0 && B <= 65535, "coco_rle: at most 65535 images per call");
  YB_REQUIRE(runs_cap >= 0 && chars_cap >= 0, "coco_rle: negative capacity");
  int max_n = 0, max_w = 0;
  int64_t rows = 0;
  for (int b = 0; b < B; ++b) {
    const yb_post_item& it = h_items[b];
    YB_REQUIRE(it.n >= 0 && it.out_h > 0 && it.out_w > 0, "coco_rle: bad sizes");
    YB_REQUIRE((int64_t)it.out_h * it.out_w <= (1ll << 28), "coco_rle: at most 2^28 pixels per image");
    rows += it.n;
    if (it.n == 0) continue;
    max_n = std::max(max_n, it.n);
    max_w = std::max(max_w, it.out_w);
  }
  YB_REQUIRE(rows < (1ll << 31), "coco_rle: too many rows");
  if (max_n == 0) {
    YB_CHECK_CUDA(cudaMemsetAsync(need, 0, 2 * sizeof(int64_t), stream));
    return;
  }
  YB_REQUIRE(k % 4 == 0 && k <= 128 && ph > 0 && pw > 0, "coco_rle: mask_dim must be a multiple of 4 and <= 128");
  // one thread per output column of a chunk; the staging buffer holds, for any image, the prototype rows (at most ph)
  // times the columns a chunk of NT output columns and its predecessor interpolate from (at most scale_w * NT + 4, and
  // pw).  Halve the chunk until that fits in 200 KB.
  int threads = std::min(CR_MAX_THREADS, ceil_div(max_w, 32) * 32);
  int64_t sig_cap = 0;
  for (;;) {
    sig_cap = 0;
    for (int b = 0; b < B; ++b) {
      const yb_post_item& it = h_items[b];
      if (it.n == 0) continue;
      sig_cap = std::max<int64_t>(sig_cap, (int64_t)ph * staged_cols(threads, pw, it.out_w));
    }
    if (sig_cap * 4 <= 200 * 1024 || threads == 32) break;
    threads /= 2;
  }
  YB_REQUIRE(sig_cap * 4 <= 200 * 1024, "coco_rle: prototypes too large for the shared-memory staging buffer");
  const size_t smem = (size_t)sig_cap * sizeof(float);
  if (smem + coco_rle_static_smem() > 48 * 1024)
    YB_CHECK_CUDA(cudaFuncSetAttribute(coco_rle_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  YB_CHECK_CUDA(cudaMemsetAsync(need, 0, 2 * sizeof(int64_t), stream));   // the rows' reservation counters
  const CocoOut o{runs, runs_cap, chars, chars_cap, row_off, row_len, reinterpret_cast<unsigned long long*>(need)};
  coco_rle_kernel<<<dim3(max_n, B), threads, smem, stream>>>(d_items, ph, pw, k, crop, o);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

}  // namespace yb
