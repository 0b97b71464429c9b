// eval.py's mAP bookkeeping (prep_metrics' matching loop, APDataObject.get_ap; eval.py:386-581) on the GPU.
//
//   eval_match : one CTA per image (yb_eval_match's one image, or every image of a yb_eval_match_list table).  The two stable score orders (eval.py:445-446) are ranked by counting, then one
//                warp per (class with detections, IoU threshold, box|mask) job replays the greedy matching loop
//                (eval.py:458-509) over that class's detections in rank order.  Every detection leaves one record
//                per (type, threshold) at slot [type][thr][rank] of the image's 2*T*n-record slot: fp32 score and
//                tag = 2 * cell + is_true, cell = (type*T + thr)*C + class, or -1 when it hit a crowd (not pushed).
//                Laid out this way a buffer of slots in image order IS the reference's push order of every cell.
//                The image's non-crowd ground-truth counts go to counts[C] (add_gt_positives).
//   eval_ap    : once at the end.  Records sorted stably by (cell, score descending) with an LSD radix sort (ties keep
//                push order, as Python's stable list.sort does), then one CTA per cell computes get_ap (eval.py:533-581)
//                in double: only the true positives move the smoothed precision-recall curve, so each TP t at sorted
//                position k contributes t / (k+1) to the first of the 101 recall bars it reaches, a suffix max over
//                the bars is the smoothed precision, and one thread sums the bars in order as Python's sum() does
//                (CPython 3.12 and later: Neumaier-compensated for floats).
//
// Limits (checked, YB_ERR_INVALID beyond them; COCO needs n <= 100, g and crowd well under 100, T = 10, C = 80):
// n, g, crowd <= 1024, 1 <= T <= 32, 1 <= C <= 2048, total records < 2^31.  A detection class outside [0, C) gets an
// "ignored" record and sets bit 0 of the error word, a ground-truth class outside it bit 1; the caller reads the word.
#include <cub/cub.cuh>

#include "kernels.cuh"

namespace yb {

namespace {

constexpr int MATCH_THREADS = 256;
constexpr int MATCH_WARPS = MATCH_THREADS / 32;
constexpr int AP_THREADS = 256;
constexpr int AP_BARS = 101;

__global__ void __launch_bounds__(MATCH_THREADS)
eval_match_kernel(EvalMatchSrc s) {
  __shared__ int s_cls[EVAL_MAX_DETS];
  __shared__ int s_rank_box[EVAL_MAX_DETS], s_rank_mask[EVAL_MAX_DETS];
  __shared__ int s_ord_box[EVAL_MAX_DETS], s_ord_mask[EVAL_MAX_DETS];
  __shared__ int s_gt_cls[EVAL_MAX_GT], s_crowd_cls[EVAL_MAX_GT];
  __shared__ int s_first[EVAL_MAX_CLASSES];   // lowest detection index of each class (n = none)
  __shared__ int s_jobs[EVAL_MAX_DETS];       // the classes with detections
  __shared__ uint32_t s_used[MATCH_WARPS][EVAL_MAX_GT / 32];
  __shared__ int s_njobs;
  const yb_eval_match_item a = s.table ? s.table[blockIdx.x] : s.one;
  const int n = a.n, g = a.g, nc = a.num_crowd, C = s.C, T = s.T;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (n == 0) return;   // eval.py:405-406: an image without detections adds nothing, not even its ground truths
  float* const rec_score = s.rec_score + a.rec_offset;
  int32_t* const rec_tag = s.rec_tag + a.rec_offset;

  for (int c = tid; c < C; c += MATCH_THREADS) s_first[c] = n;
  for (int j = tid; j < g; j += MATCH_THREADS) {
    const int c = a.gt_cls[j];
    s_gt_cls[j] = c;
    if (c >= 0 && c < C) atomicAdd(reinterpret_cast<unsigned long long*>(s.counts + c), 1ull);   // add_gt_positives
    else atomicOr(s.err, 2);
  }
  for (int j = tid; j < nc; j += MATCH_THREADS) s_crowd_cls[j] = a.crowd_cls[j];
  if (tid == 0) s_njobs = 0;
  __syncthreads();
  for (int i = tid; i < n; i += MATCH_THREADS) {
    const long long c = a.cls[i];
    const bool ok = c >= 0 && c < C;
    s_cls[i] = ok ? (int)c : -1;
    if (ok) atomicMin(&s_first[c], i);
    else atomicOr(s.err, 1);
  }
  // box_indices = sorted(range(n), key=-box_score): a stable sort, so rank(i) = #{j : s_j > s_i or (s_j == s_i, j < i)}
  for (int i = tid; i < n; i += MATCH_THREADS) {
    const float si = a.box_score[i];
    int r = 0;
    for (int j = 0; j < n; ++j) {
      const float sj = a.box_score[j];
      r += (sj > si) || (sj == si && j < i);
    }
    s_rank_box[i] = r;
    s_ord_box[r] = i;
  }
  __syncthreads();
  // mask_indices = sorted(box_indices, key=-mask_score): ties keep the box order
  for (int i = tid; i < n; i += MATCH_THREADS) {
    const float si = a.mask_score[i];
    const int bi = s_rank_box[i];
    int r = 0;
    for (int j = 0; j < n; ++j) {
      const float sj = a.mask_score[j];
      r += (sj > si) || (sj == si && s_rank_box[j] < bi);
    }
    s_rank_mask[i] = r;
    s_ord_mask[r] = i;
  }
  __syncthreads();
  // the classes with detections, as a job list (order is irrelevant: jobs write disjoint records)
  for (int i = tid; i < n; i += MATCH_THREADS) {
    const int c = s_cls[i];
    if (c >= 0 && s_first[c] == i) s_jobs[atomicAdd(&s_njobs, 1)] = c;
  }
  __syncthreads();
  const int njobs = s_njobs * T * 2;
  const int64_t n64 = n;
  for (int job = warp; job < njobs; job += MATCH_WARPS) {
    const int type = job & 1, thr = (job >> 1) % T, c = s_jobs[(job >> 1) / T];
    const double th = s.thr[thr];
    const float* iou = type ? a.mask_iou : a.box_iou;
    const float* ciou = type ? a.crowd_mask_iou : a.crowd_box_iou;
    const float* score = type ? a.mask_score : a.box_score;
    const int* ord = type ? s_ord_mask : s_ord_box;
    uint32_t* used = s_used[warp];
    for (int w = lane; w < EVAL_MAX_GT / 32; w += 32) used[w] = 0u;
    __syncwarp();
    const int tag_base = 2 * ((type * T + thr) * C + c);
    float* out_score = rec_score + (int64_t)(type * T + thr) * n64;
    int32_t* out_tag = rec_tag + (int64_t)(type * T + thr) * n64;
    for (int r0 = 0; r0 < n; r0 += 32) {
      const int r = r0 + lane;
      const int i_l = r < n ? ord[r] : 0;
      uint32_t mine = __ballot_sync(0xffffffffu, r < n && s_cls[i_l] == c);
      while (mine) {
        const int l = __ffs(mine) - 1;
        mine &= mine - 1;
        const int i = __shfl_sync(0xffffffffu, i_l, l);
        // max IoU over the unused ground truths of the class, `iou > max_iou_found` from max_iou_found = thr:
        // the largest IoU strictly above thr (compared as doubles), the lowest j among equal ones; NaN never matches
        float best = 0.f;
        int bj = -1;
        for (int j = lane; j < g; j += 32) {
          if (s_gt_cls[j] != c || ((used[j >> 5] >> (j & 31)) & 1u)) continue;
          const float v = iou[(int64_t)i * g + j];
          if ((double)v > th && (bj < 0 || v > best)) {
            best = v;
            bj = j;
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float ob = __shfl_xor_sync(0xffffffffu, best, o);
          const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
          if (oj >= 0 && (bj < 0 || ob > best || (ob == best && oj < bj))) {
            best = ob;
            bj = oj;
          }
        }
        bool crowd = false;
        if (bj < 0) {   // only an unmatched detection is tested against the crowd (eval.py:490-503)
          bool hit = false;
          for (int j = lane; j < nc; j += 32)
            hit |= s_crowd_cls[j] == c && (double)ciou[(int64_t)i * nc + j] > th;
          crowd = __any_sync(0xffffffffu, hit);
        }
        if (lane == 0) {
          if (bj >= 0) used[bj >> 5] |= 1u << (bj & 31);
          const int rk = type ? s_rank_mask[i] : s_rank_box[i];
          out_score[rk] = score[i];
          out_tag[rk] = bj >= 0 ? tag_base + 1 : (crowd ? -1 : tag_base);
        }
        __syncwarp();
      }
    }
  }
  // detections with a class outside [0, C): an "ignored" record in every (type, threshold), and the error word is set
  for (int idx = tid; idx < 2 * T * n; idx += MATCH_THREADS) {
    const int i = idx % n, tt = idx / n;
    if (s_cls[i] < 0) {
      const int rk = (tt >= T) ? s_rank_mask[i] : s_rank_box[i];
      rec_score[(int64_t)tt * n64 + rk] = 0.f;
      rec_tag[(int64_t)tt * n64 + rk] = -1;
    }
  }
}

// ---- AP step -----------------------------------------------------------------------------------------------------
// key = cell << 32 | ~(order-preserving bits of the score): ascending keys = ascending cell, descending score.
// -0.0 is made +0.0 (they compare equal in Python).  Crowd hits get the cell past the last one.
__global__ void __launch_bounds__(256)
eval_keys_kernel(const float* __restrict__ score, const int32_t* __restrict__ tag, int64_t R, uint32_t ncells,
                 unsigned long long* __restrict__ keys, uint8_t* __restrict__ tp) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x) {
    const int32_t t = tag[r];
    uint32_t u = __float_as_uint(score[r]);
    if (u == 0x80000000u) u = 0u;
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);   // ascending float order
    const uint32_t cell = t < 0 ? ncells : (uint32_t)(t >> 1);
    keys[r] = ((unsigned long long)cell << 32) | (unsigned long long)(~u);
    tp[r] = (uint8_t)(t >= 0 ? (t & 1) : 0);
  }
}

__global__ void __launch_bounds__(256)
eval_bounds_kernel(const unsigned long long* __restrict__ keys, int64_t R, uint32_t ncells, int64_t* __restrict__ begin,
                   int64_t* __restrict__ end) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t c = (uint32_t)(keys[r] >> 32);
    if (c >= ncells) continue;
    if (r == 0 || (uint32_t)(keys[r - 1] >> 32) != c) begin[c] = r;
    if (r == R - 1 || (uint32_t)(keys[r + 1] >> 32) != c) end[c] = r + 1;
  }
}

// One CTA per cell (type, thr, class): APDataObject.get_ap on the cell's sorted true/false flags.
//   precision_k = tp_k / (k+1), recall_k = tp_k / G (doubles); bar b (x_b = b / 100.0) reads the smoothed precision
//   max_{k >= idx_b} precision_k at idx_b = first k with recall_k >= x_b, or 0 past the end.
// recall_k >= x_b  <=>  tp_k >= m_b, the smallest integer with m_b / G >= x_b (division is monotone), so idx_b is the
// position of the m_b-th TP (0 when m_b == 0).  Precision only rises at a TP, hence the smoothed value at idx_b is the
// max of t / (pos_t + 1) over the TPs t >= max(m_b, 1): TP t goes to the last bar b with m_b <= t, and a suffix max
// over the bars gives every bar's value.  The 101 bars are summed in order by one thread, as Python's sum() does.
__global__ void __launch_bounds__(AP_THREADS)
eval_ap_kernel(const uint8_t* __restrict__ tp, const int64_t* __restrict__ begin, const int64_t* __restrict__ end,
               const int64_t* __restrict__ counts, int C, double* __restrict__ ap, uint8_t* __restrict__ nonempty) {
  __shared__ long long s_m[AP_BARS];
  __shared__ unsigned long long s_bar[AP_BARS];   // bit patterns of non-negative doubles order like the doubles
  __shared__ int s_warp[AP_THREADS / 32];
  const int cell = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const long long G = counts[cell % C];
  const int64_t b0 = begin[cell], e = end[cell];
  if (tid == 0) nonempty[cell] = (e > b0 || G != 0) ? 1 : 0;
  if (G <= 0) {   // `if self.num_gt_positives == 0: return 0`
    if (tid == 0) ap[cell] = 0.0;
    return;
  }
  const double Gd = (double)G;
  if (tid < AP_BARS) {
    const double x = (double)tid / 100.0;
    long long m = (long long)ceil(x * Gd);
    if (m < 0) m = 0;
    while (m > 0 && (double)(m - 1) / Gd >= x) --m;
    while ((double)m / Gd < x) ++m;
    s_m[tid] = m;
    s_bar[tid] = 0ull;
  }
  __syncthreads();
  long long carry = 0;
  for (int64_t base = b0; base < e; base += AP_THREADS) {
    const int64_t k = base + tid;
    const int f = k < e ? (int)tp[k] : 0;
    int inc = f;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += v;
    }
    if (lane == 31) s_warp[wid] = inc;
    __syncthreads();
    int woff = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < AP_THREADS / 32; ++w) {
      const int c = s_warp[w];
      woff += w < wid ? c : 0;
      tot += c;
    }
    if (f) {
      const long long t = carry + woff + inc;
      const double prec = (double)t / (double)(k - b0 + 1);
      int lo = 0, hi = AP_BARS - 1;   // last bar with m_b <= t (m_0 == 0 <= t)
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (s_m[mid] <= t) lo = mid;
        else hi = mid - 1;
      }
      atomicMax(&s_bar[lo], (unsigned long long)__double_as_longlong(prec));
    }
    carry += tot;
    __syncthreads();   // s_warp is rewritten by the next chunk
  }
  if (tid == 0) {
    unsigned long long run = 0ull;   // suffix max, in place
    for (int b = AP_BARS - 1; b >= 0; --b) {
      run = s_bar[b] > run ? s_bar[b] : run;
      s_bar[b] = run;
    }
    // sum(y_range): CPython (3.12 on) adds floats with Neumaier's compensation and adds the compensation at the end
    double s = 0.0, comp = 0.0;
    for (int b = 0; b < AP_BARS; ++b) {
      const double x = __longlong_as_double((long long)s_bar[b]);
      const double t = s + x;
      comp += fabs(s) >= fabs(x) ? (s - t) + x : (x - t) + s;
      s = t;
    }
    if (comp != 0.0 && isfinite(comp)) s += comp;
    ap[cell] = s / (double)AP_BARS;
  }
}

inline int grid_for(int64_t total, int block) {
  int64_t g = (total + block - 1) / block;
  const int64_t cap = 132 * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

inline int bits_for(uint32_t v) {
  int b = 0;
  while (b < 32 && (v >> b) != 0u) ++b;
  return b;
}

struct ApWork {
  unsigned long long *keys_in, *keys_out;
  uint8_t *tp_in, *tp_out;
  int64_t *begin, *end;
  void* cub_tmp;
  size_t cub_bytes;
  size_t total;
};

inline size_t align_up(size_t v) { return (v + 255) & ~(size_t)255; }

ApWork eval_ap_layout(int64_t R, int T, int C, void* base) {
  ApWork w{};
  const int ncells = 2 * T * C;
  const int end_bit = 32 + bits_for((uint32_t)ncells);
  size_t cub_bytes = 0;
  YB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const unsigned long long*)nullptr,
                                                (unsigned long long*)nullptr, (const uint8_t*)nullptr, (uint8_t*)nullptr,
                                                (int)R, 0, end_bit));
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? (char*)base + off : nullptr;
    off += align_up(bytes);
    return (void*)p;
  };
  w.keys_in = (unsigned long long*)take(sizeof(unsigned long long) * R);
  w.keys_out = (unsigned long long*)take(sizeof(unsigned long long) * R);
  w.tp_in = (uint8_t*)take(R);
  w.tp_out = (uint8_t*)take(R);
  w.begin = (int64_t*)take(sizeof(int64_t) * 2 * (size_t)ncells);
  w.end = w.begin ? w.begin + ncells : nullptr;
  w.cub_tmp = take(cub_bytes);
  w.cub_bytes = cub_bytes;
  w.total = off;
  return w;
}

}  // namespace

void eval_check_limits(int n, int g, int num_crowd, int T, int C) {
  YB_REQUIRE(n >= 0 && n <= EVAL_MAX_DETS, "eval_match: at most 1024 detections per image");
  YB_REQUIRE(g >= 0 && g <= EVAL_MAX_GT, "eval_match: at most 1024 ground truths per image");
  YB_REQUIRE(num_crowd >= 0 && num_crowd <= EVAL_MAX_GT, "eval_match: at most 1024 crowd ground truths per image");
  YB_REQUIRE(T >= 1 && T <= EVAL_MAX_THRESHOLDS, "eval: 1 to 32 IoU thresholds");
  YB_REQUIRE(C >= 1 && C <= EVAL_MAX_CLASSES, "eval: 1 to 2048 classes");
}

void launch_eval_match(const EvalMatchSrc& src, const yb_eval_match_item* h_items, int B, cudaStream_t stream,
                       LaunchCounter* lc) {
  YB_REQUIRE(B >= 0 && (B == 0 || h_items), "eval_match: bad image list");
  bool any = false;
  for (int b = 0; b < B; ++b) {
    eval_check_limits(h_items[b].n, h_items[b].g, h_items[b].num_crowd, src.T, src.C);
    YB_REQUIRE(h_items[b].rec_offset >= 0, "eval_match: negative record offset");
    any |= h_items[b].n > 0;
  }
  if (!any) return;   // eval.py:405-406: an image without detections adds nothing, not even its ground truths
  eval_match_kernel<<<B, MATCH_THREADS, 0, stream>>>(src);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

size_t eval_ap_workspace_bytes(int64_t R, int T, int C) {
  YB_REQUIRE(R >= 0 && R < (1ll << 31) - 1, "eval_ap: fewer than 2^31 records");
  eval_check_limits(0, 0, 0, T, C);
  return eval_ap_layout(R, T, C, nullptr).total;
}

void launch_eval_ap(const float* rec_score, const int32_t* rec_tag, int64_t R, const int64_t* counts, int T, int C,
                    void* work, size_t work_bytes, double* ap, uint8_t* nonempty, cudaStream_t stream, LaunchCounter* lc) {
  YB_REQUIRE(work_bytes >= eval_ap_workspace_bytes(R, T, C), "eval_ap: workspace too small");
  const int ncells = 2 * T * C;
  ApWork w = eval_ap_layout(R, T, C, work);
  YB_CHECK_CUDA(cudaMemsetAsync(w.begin, 0, sizeof(int64_t) * 2 * (size_t)ncells, stream));
  if (R > 0) {
    eval_keys_kernel<<<grid_for(R, 256), 256, 0, stream>>>(rec_score, rec_tag, R, (uint32_t)ncells, w.keys_in, w.tp_in);
    YB_CHECK_LAUNCH();
    size_t cub_bytes = w.cub_bytes;
    YB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.cub_tmp, cub_bytes, w.keys_in, w.keys_out, w.tp_in, w.tp_out, (int)R,
                                                  0, 32 + bits_for((uint32_t)ncells), stream));
    eval_bounds_kernel<<<grid_for(R, 256), 256, 0, stream>>>(w.keys_out, R, (uint32_t)ncells, w.begin, w.end);
    YB_CHECK_LAUNCH();
    if (lc) lc->n += 3;
  }
  eval_ap_kernel<<<ncells, AP_THREADS, 0, stream>>>(w.tp_out, w.begin, w.end, counts, C, ap, nonempty);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

}  // namespace yb
