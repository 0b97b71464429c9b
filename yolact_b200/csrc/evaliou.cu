// prep_metrics' IoU caches (eval.py:431-445: _bbox_iou, _mask_iou and their crowd forms) for a list of images straight
// from the detections: the masks yb_postprocess would write are formed word by word on the ground truth's bit layout
// and never stored.
//
//   eval_iou_kernel : one CTA per (detection row, image) (blockIdx.x = row, blockIdx.y = image of the yb_eval_iou_item
//                     table).  Box IoUs: box_jaccard of the row's pixel box (int64 -> fp32, as .float() converts it)
//                     against every ground-truth box.  Mask IoUs: only the output pixels inside window_out_bounds of
//                     the row's crop window, columns [xa, xb) x rows [ya, yb), can be set.  For each chunk of up to 32
//                     words of columns, StagedMask stages the cropped sigmoid values those columns read; then each warp
//                     takes rows of the chunk, forms each 32-pixel word of the row with a ballot (zero outside the
//                     window), keeps word i in lane i, and adds popc(word & gt_word) of every ground truth to its own
//                     per-warp counters (one warp reduction per ground truth and row).  The detection's area is the sum
//                     of popc(word); the non-crowd ground truths' areas are popcounts over their whole masks.
//
// The pixels are yb_postprocess's (same functions, same crop-before-upsample order, zero outside the window), so the
// intersections and areas are the integers yb_mask_iou counts on yb_postprocess's bits, and mask_iou_counts divides
// them as mask_iou_bits_kernel does: every cache is bit-identical, 0 / 0 = NaN included.
#include <algorithm>
#include "kernels.cuh"
#include "staged_mask.cuh"

namespace yb {

namespace {

constexpr int EI_THREADS = 256;
constexpr int EI_WARPS = EI_THREADS / 32;
constexpr int EI_MAX_CHUNK_WORDS = 32;   // one word per lane

// dynamic shared memory: sig [sig_cap] floats | acc [EI_WARPS][g_all] | gt_area [g_all]
__global__ void __launch_bounds__(EI_THREADS)
eval_iou_kernel(const yb_eval_iou_item* __restrict__ items, int ph, int pw, int k, int crop, int chunk_words,
                int sig_cap) {
  __shared__ yb_eval_iou_item it;
  __shared__ unsigned s_area[EI_WARPS];
  extern __shared__ float smem[];
  const int b = blockIdx.y, d = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) it = items[b];
  __syncthreads();
  const int ga = it.g_all;
  if (d >= it.n || ga == 0) return;   // uniform
  const int h = it.out_h, w = it.out_w, wpr = (w + 31) >> 5, nc = it.num_crowd, g = ga - nc;
  const int64_t plane = (int64_t)h * wpr;
  float* sig = smem;
  unsigned* acc = reinterpret_cast<unsigned*>(smem + sig_cap);
  unsigned* gt_area = acc + EI_WARPS * ga;

  // box IoUs: jaccard(boxes_px.float(), gt_boxes)
  const int64_t* bp = it.boxes_px + (size_t)d * 4;
  const float4 A = make_float4((float)bp[0], (float)bp[1], (float)bp[2], (float)bp[3]);
  for (int j = tid; j < ga; j += EI_THREADS) {
    const float* gb = it.gt_boxes + (size_t)j * 4;
    const float4 G = make_float4(gb[0], gb[1], gb[2], gb[3]);
    if (j < g) it.box_iou[(int64_t)d * g + j] = box_jaccard(A, G, 0);
    else it.crowd_box_iou[(int64_t)d * nc + (j - g)] = box_jaccard(A, G, 1);
  }
  for (int i = tid; i < EI_WARPS * ga; i += EI_THREADS) acc[i] = 0u;
  // the non-crowd ground truths' areas (a crowd IoU divides by the detection's area only)
  for (int j = warp; j < g; j += EI_WARPS) {
    const uint32_t* p = it.gt_bits + j * plane;
    unsigned c = 0;
    for (int64_t q = lane; q < plane; q += 32) c += __popc(__ldg(p + q));
    c = __reduce_add_sync(0xffffffffu, c);
    if (lane == 0) gt_area[j] = c;
  }
  __syncthreads();   // acc is zero before any warp adds to it

  StagedMask px;
  int xa, xb, ya, yb;
  px.init(it.proto, it.coef, it.box, d, crop, ph, pw, k, h, w, sig, &xa, &xb, &ya, &yb);
  unsigned area = 0;   // this lane's share of the detection's area
  unsigned* my_acc = acc + warp * ga;
  const int wa = xa >> 5, wb = (xb + 31) >> 5;   // xa == xb == 0 for an empty window: no chunk
  for (int w0 = wa; w0 < wb; w0 += chunk_words) {   // uniform
    const int w1 = min(w0 + chunk_words, wb);
    px.chunk(max(w0 * 32, xa), min(w1 * 32, xb));
    const bool in = w0 + lane < w1;   // lane i keeps word w0 + i of the row
    for (int y = ya + warp; y < yb; y += EI_WARPS) {
      uint32_t mine = 0u;
      for (int i = 0; i < w1 - w0; ++i) {
        const int x = (w0 + i) * 32 + lane;
        const uint32_t word = __ballot_sync(0xffffffffu, x >= xa && x < xb && px(y, x));
        if (lane == i) mine = word;
      }
      area += __popc(mine);
      if (!__any_sync(0xffffffffu, mine != 0u)) continue;   // nothing set in this row of the chunk
      const uint32_t* gp = it.gt_bits + (int64_t)y * wpr + w0 + lane;
      for (int j = 0; j < ga; ++j) {
        const uint32_t gw = in ? __ldg(gp + j * plane) : 0u;
        const unsigned v = __reduce_add_sync(0xffffffffu, (unsigned)__popc(mine & gw));
        if (lane == 0) my_acc[j] += v;
      }
    }
  }
  area = __reduce_add_sync(0xffffffffu, area);
  if (lane == 0) s_area[warp] = area;
  __syncthreads();
  unsigned fa = 0;
#pragma unroll
  for (int i = 0; i < EI_WARPS; ++i) fa += s_area[i];
  for (int j = tid; j < ga; j += EI_THREADS) {
    unsigned inter = 0;
#pragma unroll
    for (int i = 0; i < EI_WARPS; ++i) inter += acc[i * ga + j];
    if (j < g) it.mask_iou[(int64_t)d * g + j] = mask_iou_counts(inter, fa, gt_area[j], 0);
    else it.crowd_mask_iou[(int64_t)d * nc + (j - g)] = mask_iou_counts(inter, fa, 0u, 1);
  }
}

size_t eval_iou_static_smem() {
  static const size_t bytes = [] {
    cudaFuncAttributes a{};
    YB_CHECK_CUDA(cudaFuncGetAttributes(&a, eval_iou_kernel));
    return a.sharedSizeBytes;
  }();
  return bytes;
}

}  // namespace

void launch_eval_iou(const yb_eval_iou_item* d_items, const yb_eval_iou_item* h_items, int B, int ph, int pw, int k,
                     int crop, cudaStream_t stream, LaunchCounter* lc) {
  YB_REQUIRE(B >= 0 && B <= 65535, "eval_iou: at most 65535 images per call");
  int max_n = 0, g_cap = 0;
  for (int b = 0; b < B; ++b) {
    const yb_eval_iou_item& it = h_items[b];
    YB_REQUIRE(it.n >= 0 && it.n <= EVAL_MAX_DETS && it.out_h > 0 && it.out_w > 0, "eval_iou: bad sizes");
    YB_REQUIRE(it.num_crowd >= 0 && it.num_crowd <= it.g_all && it.g_all <= 2 * EVAL_MAX_GT, "eval_iou: bad ground truth");
    if (it.n == 0 || it.g_all == 0) continue;
    max_n = std::max(max_n, it.n);
    g_cap = std::max(g_cap, it.g_all);
  }
  if (max_n == 0) return;   // no image has both detections and ground truth: every cache is empty
  YB_REQUIRE(k % 4 == 0 && k <= 128 && ph > 0 && pw > 0, "eval_iou: mask_dim must be a multiple of 4 and <= 128");
  // staging buffer: ph prototype rows times the columns a chunk of 32 * chunk_words output columns and its predecessor
  // read (as coco_rle's); halve the chunk until it fits beside the per-warp counters
  const size_t fixed = (size_t)(EI_WARPS + 1) * g_cap * sizeof(unsigned);
  const size_t budget = 220 * 1024 - eval_iou_static_smem();
  int chunk_words = EI_MAX_CHUNK_WORDS;
  int64_t sig_cap = 0;
  for (;;) {
    sig_cap = 0;
    for (int b = 0; b < B; ++b) {
      const yb_eval_iou_item& it = h_items[b];
      if (it.n == 0 || it.g_all == 0) continue;
      sig_cap = std::max<int64_t>(sig_cap, (int64_t)ph * staged_cols(32 * chunk_words, pw, it.out_w));
    }
    if ((size_t)sig_cap * sizeof(float) + fixed <= budget || chunk_words == 1) break;
    chunk_words /= 2;
  }
  const size_t smem = (size_t)sig_cap * sizeof(float) + fixed;
  YB_REQUIRE(smem <= budget, "eval_iou: prototypes too large for the shared-memory staging buffer");
  if (smem + eval_iou_static_smem() > 48 * 1024)
    YB_CHECK_CUDA(cudaFuncSetAttribute(eval_iou_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  eval_iou_kernel<<<dim3(max_n, B), EI_THREADS, smem, stream>>>(d_items, ph, pw, k, crop, chunk_words, (int)sig_cap);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

}  // namespace yb
