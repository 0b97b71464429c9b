// Detect: softmax -> score threshold -> per-class top-k -> decode -> Fast NMS -> global top-k
// (plus the --fast_nms=False variant: greedy per-class NMS, trad_nms_kernel).
//
// Reference: Detect.__call__/detect/fast_nms/cc_fast_nms (layers/functions/detection.py:32-180),
// decode (layers/box_utils.py:267-312, non-yolo branch), jaccard/intersect (box_utils.py:32-80),
// F.softmax (yolact.py:674).
//
// The reference runs ~15 ATen launches with host syncs on boolean indexing; here it is three
// launches with no host involvement:
//   K1 detect_candidates : [P,C] logits/probs tile -> softmax -> max fg score > conf_thresh ->
//                          compacted class-major score matrix scoresT[c][m] + prior index list.
//   K2 class_nms         : one CTA per (class, image): exact top-k by radix select on a 64-bit
//                          (score, ~prior) key, bitonic sort, decode, upper-triangular IoU column
//                          max, keep <= nms_thresh (suppressed boxes still suppress: detection.py:148-150).
//   K3 final_select      : one CTA per image: top max_dets of all kept (class, rank) entries,
//                          gathers box / mask coefficients / class / score.
// Ordering contract (the reference's torch.sort is unstable, SURVEY.md Appendix D.18): ties in
// score are broken by lower prior index (per class) and lower (class, rank) (final), i.e. what a
// stable sort of the reference's tensors yields.
//
// All score / box arithmetic uses round-to-nearest intrinsics so nvcc cannot contract a*b+c into
// FMA: given identical inputs the keep decisions are the reference's, up to expf's last ulp.
// Scores are ordered by their float bits, which order non-negative floats only: negative or -0.0
// "probabilities" are outside the contract (a softmax cannot produce them).  A prior with a NaN
// foreground score is no candidate, as torch.max propagates NaN into the reference's threshold test.
#include "kernels.cuh"

namespace yb {

namespace {

constexpr int K1_ROWS = 128;   // priors per CTA in K1
constexpr int K1_HEADER_BYTES = 32;   // K1's warp counts and block base, ahead of its [K1_ROWS][C] tile
constexpr int NT2 = 256;       // threads in K2 / K3
constexpr int SORT_N = 256;    // bitonic sort width (>= top_k)
constexpr int HIST_BINS = 2048;

// ---------------------------------------------------------------------------------------------
// K1
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(K1_ROWS)
detect_candidates_kernel(const float* __restrict__ conf, int64_t P, int C, int is_logits,
                         float conf_thresh, int cross_class, float* __restrict__ scoresT,
                         int32_t* __restrict__ cand_prior, int32_t* __restrict__ cand_cls,
                         int32_t* __restrict__ cand_count) {
  // all of K1's shared memory is dynamic, so the launch's size is the whole footprint
  extern __shared__ __align__(16) unsigned char k1_smem[];
  int* warp_cnt = reinterpret_cast<int*>(k1_smem);                    // [K1_ROWS / 32]
  int& s_base = warp_cnt[K1_ROWS / 32];
  float* tile = reinterpret_cast<float*>(k1_smem + K1_HEADER_BYTES);   // [K1_ROWS][C]

  const int b = blockIdx.y;
  const int64_t p0 = (int64_t)blockIdx.x * K1_ROWS;
  const int rows = (int)min((int64_t)K1_ROWS, P - p0);
  const float* src = conf + ((int64_t)b * P + p0) * C;
  for (int i = threadIdx.x; i < rows * C; i += K1_ROWS) tile[i] = src[i];
  __syncthreads();

  const int t = threadIdx.x;
  float* row = tile + t * C;
  bool keep = false;
  float best = -1.f;
  int best_c = 0;
  if (t < rows) {
    if (is_logits) {
      float m = row[0];
      for (int c = 1; c < C; ++c) m = fmaxf(m, row[c]);
      float s = 0.f;
      for (int c = 0; c < C; ++c) {
        float e = expf(__fsub_rn(row[c], m));
        row[c] = e;
        s = __fadd_rn(s, e);
      }
      for (int c = 0; c < C; ++c) row[c] = __fdiv_rn(row[c], s);
    }
    // max over foreground classes (detection.py:83-84); first max wins like torch.max, and a NaN
    // anywhere makes torch.max NaN, which fails `> conf_thresh`
    best = row[1];
    best_c = 0;
    bool nan = best != best;
    for (int c = 2; c < C; ++c) {
      const float v = row[c];
      nan |= v != v;
      if (v > best) {
        best = v;
        best_c = c - 1;
      }
    }
    keep = !nan && best > conf_thresh;
  }
  // block-level ordered compaction
  unsigned bal = __ballot_sync(0xffffffffu, keep);
  const int lane = t & 31, wid = t >> 5;
  if (lane == 0) warp_cnt[wid] = __popc(bal);
  __syncthreads();
  int woff = 0, total = 0;
#pragma unroll
  for (int w = 0; w < K1_ROWS / 32; ++w) {
    if (w < wid) woff += warp_cnt[w];
    total += warp_cnt[w];
  }
  if (t == 0) s_base = total ? atomicAdd(&cand_count[b], total) : 0;
  __syncthreads();
  if (!keep) return;
  const int64_t slot = s_base + woff + __popc(bal & ((1u << lane) - 1u));
  cand_prior[(int64_t)b * P + slot] = (int32_t)(p0 + t);
  if (cross_class) {
    scoresT[(int64_t)b * (C - 1) * P + slot] = best;
    cand_cls[(int64_t)b * P + (p0 + t)] = best_c;  // indexed by PRIOR (K2 only knows the prior)
  } else {
    float* dst = scoresT + (int64_t)b * (C - 1) * P + slot;
    for (int c = 1; c < C; ++c) dst[(int64_t)(c - 1) * P] = row[c];
  }
}

// ---------------------------------------------------------------------------------------------
// block-wide helpers (NT2 threads)
// ---------------------------------------------------------------------------------------------
// Exclusive prefix sum of one int per thread; returns (exclusive, total).
__device__ __forceinline__ int block_excl_scan(int v, int* s_warp /*[NT2/32]*/, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int n = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += n;
  }
  __syncthreads();  // protect s_warp reuse
  if (lane == 31) s_warp[wid] = inc;
  __syncthreads();
  int woff = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < NT2 / 32; ++w) {
    int c = s_warp[w];
    if (w < wid) woff += c;
    tot += c;
  }
  *total = tot;
  return woff + inc - v;
}

struct SelectScratch {
  uint32_t hist[HIST_BINS];
  int warp[NT2 / 32];
  unsigned long long prefix;
  int need;
  int done;
  int sel_count;
};

// Exact top-K (by unique 64-bit key, larger is better) of n virtual items.  key(i) may return 0
// for "absent" items; absent items must never be needed (K <= number of present items).
// Writes the K selected keys (unordered) to sel[0..K) and zero-fills sel[K..SORT_N).
template <typename KeyFn>
__device__ void block_select_topk(KeyFn key, int n, int K, unsigned long long* sel, SelectScratch* sc) {
  const int tid = threadIdx.x;
  for (int i = tid; i < SORT_N; i += NT2) sel[i] = 0ull;
  if (tid == 0) {
    sc->prefix = 0ull;
    sc->need = K;
    sc->done = 0;
    sc->sel_count = 0;
  }
  __syncthreads();
  int final_shift = 0;
  if (n > K) {
    const int shifts[6] = {53, 42, 32, 21, 10, 0};
    const int bitsv[6] = {11, 11, 10, 11, 11, 10};
    for (int pass = 0; pass < 6; ++pass) {
      const int shift = shifts[pass], bits = bitsv[pass];
      const int nb = 1 << bits;
      for (int i = tid; i < nb; i += NT2) sc->hist[i] = 0u;
      __syncthreads();
      const unsigned long long prefix = sc->prefix;
      for (int i = tid; i < n; i += NT2) {
        unsigned long long k = key(i);
        if (k == 0ull) continue;
        bool match = (pass == 0) || ((k >> (shift + bits)) == prefix);
        if (match) atomicAdd(&sc->hist[(unsigned)(k >> shift) & (nb - 1)], 1u);
      }
      __syncthreads();
      // each thread owns `per` consecutive bins, find the bin where the running count from the
      // top crosses `need`
      const int per = nb / NT2;
      int local = 0;
      for (int j = 0; j < per; ++j) local += (int)sc->hist[tid * per + j];
      int total;
      int excl = block_excl_scan(local, sc->warp, &total);
      int above = total - excl - local;  // keys in bins owned by higher threads
      const int need = sc->need;
      __syncthreads();
      if (above < need && need <= above + local) {
        int cum = above;
        for (int j = per - 1; j >= 0; --j) {
          int h = (int)sc->hist[tid * per + j];
          if (cum + h >= need) {
            sc->prefix = (prefix << bits) | (unsigned long long)(tid * per + j);
            sc->need = need - cum;
            sc->done = (h == need - cum) ? 1 : 0;
            break;
          }
          cum += h;
        }
      }
      __syncthreads();
      final_shift = shift;
      if (sc->done) break;
    }
  } else {
    final_shift = 64;  // take everything present
  }
  const unsigned long long prefix = sc->prefix;
  for (int i = tid; i < n; i += NT2) {
    unsigned long long k = key(i);
    if (k == 0ull) continue;
    bool take = (final_shift >= 64) || ((k >> final_shift) >= prefix);
    if (take) {
      int pos = atomicAdd(&sc->sel_count, 1);
      if (pos < SORT_N) sel[pos] = k;
    }
  }
  __syncthreads();
}

// In-place descending bitonic sort of SORT_N 64-bit keys in shared memory (NT2 == SORT_N threads).
__device__ void block_sort_desc(unsigned long long* a) {
  const int tid = threadIdx.x;
  for (int size = 2; size <= SORT_N; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      int partner = tid ^ stride;
      if (partner > tid) {
        bool desc = ((tid & size) == 0);
        unsigned long long x = a[tid], y = a[partner];
        bool swap = desc ? (x < y) : (x > y);
        if (swap) {
          a[tid] = y;
          a[partner] = x;
        }
      }
    }
  }
  __syncthreads();
}

__device__ __forceinline__ float4 decode_box(const float* __restrict__ loc, const float* __restrict__ pri) {
  // box_utils.py:303-310  (variances 0.1 / 0.2;  x1 = cx - w/2;  x2 = x1 + w)
  float cx = __fadd_rn(pri[0], __fmul_rn(__fmul_rn(loc[0], 0.1f), pri[2]));
  float cy = __fadd_rn(pri[1], __fmul_rn(__fmul_rn(loc[1], 0.1f), pri[3]));
  float w = __fmul_rn(pri[2], expf(__fmul_rn(loc[2], 0.2f)));
  float h = __fmul_rn(pri[3], expf(__fmul_rn(loc[3], 0.2f)));
  float x1 = __fsub_rn(cx, __fdiv_rn(w, 2.f));
  float y1 = __fsub_rn(cy, __fdiv_rn(h, 2.f));
  return make_float4(x1, y1, __fadd_rn(x1, w), __fadd_rn(y1, h));
}

__device__ __forceinline__ float box_iou(const float4& a, const float4& b) {
  // box_utils.py:46-51, 72-79
  float iw = fmaxf(__fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)), 0.f);
  float ih = fmaxf(__fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)), 0.f);
  float inter = __fmul_rn(iw, ih);
  float area_a = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
  float area_b = __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
  float uni = __fsub_rn(__fadd_rn(area_a, area_b), inter);
  return __fdiv_rn(inter, uni);
}

// torch.max semantics: NaN propagates
__device__ __forceinline__ float nan_max(float m, float v) {
  return (m != m) ? m : ((v != v) ? v : fmaxf(m, v));
}

// ---------------------------------------------------------------------------------------------
// K2: per (class, image) Fast NMS.   CC = cross-class variant (one CTA per image, writes output).
// ---------------------------------------------------------------------------------------------
template <bool CC>
__global__ void __launch_bounds__(NT2)
class_nms_kernel(const float* __restrict__ scoresT, const int32_t* __restrict__ cand_prior,
                 const int32_t* __restrict__ cand_cls, const int32_t* __restrict__ cand_count,
                 const float* __restrict__ loc, const float* __restrict__ priors,
                 const float* __restrict__ coef, int64_t P, int C, int mask_dim, int top_k,
                 float nms_thresh,
                 float second_thresh,   // fast_nms(second_threshold=True): keep only score > conf_thresh; -inf = off
                 // per-class pool (not CC)
                 float* __restrict__ pool_score, int32_t* __restrict__ pool_prior,
                 float* __restrict__ pool_box, int32_t* __restrict__ pool_n,
                 // direct outputs (CC)
                 int max_out, float* __restrict__ out_box, float* __restrict__ out_coef,
                 int64_t* __restrict__ out_cls, float* __restrict__ out_score,
                 int32_t* __restrict__ out_count) {
  __shared__ unsigned long long sel[SORT_N];
  __shared__ SelectScratch sc;
  __shared__ float4 sbox[SORT_N];
  __shared__ int s_warp[NT2 / 32];

  const int c = blockIdx.x;  // class row (0-based over foreground); 0 for CC
  const int b = blockIdx.y;
  const int tid = threadIdx.x;
  const int M = cand_count[b];
  // CC: output rows [n, max_out) are zero, as final_select_kernel leaves them (max_out <= NT2)
  auto cc_zero_rows_from = [&](int n) {
    if (tid >= n && tid < max_out) {
      const int64_t o = (int64_t)b * max_out + tid;
      reinterpret_cast<float4*>(out_box)[o] = make_float4(0.f, 0.f, 0.f, 0.f);
      out_score[o] = 0.f;
      out_cls[o] = 0;
      for (int k = 0; k < mask_dim; ++k) out_coef[o * mask_dim + k] = 0.f;
    }
  };
  if (M == 0) {
    if (CC) {
      cc_zero_rows_from(0);
      if (tid == 0) out_count[b] = 0;
    } else if (tid == 0) {
      pool_n[b * (C - 1) + c] = 0;
    }
    return;
  }
  const float* sc_row = scoresT + ((int64_t)b * (C - 1) + c) * P;
  const int32_t* cp = cand_prior + (int64_t)b * P;
  const int K = min(top_k, M);

  auto keyfn = [&](int i) -> unsigned long long {
    unsigned hi = __float_as_uint(sc_row[i]);
    unsigned lo = 0xFFFFFFFFu - (unsigned)cp[i];
    // a present item never yields key 0: prior < 2^31 so lo >= 0x80000000
    return ((unsigned long long)hi << 32) | (unsigned long long)lo;
  };
  block_select_topk(keyfn, M, K, sel, &sc);
  block_sort_desc(sel);

  // decode the K candidates (rank order)
  const unsigned long long mykey = sel[tid];
  const bool valid = tid < K;
  const int prior = valid ? (int)(0xFFFFFFFFu - (unsigned)(mykey & 0xFFFFFFFFull)) : 0;
  const float score = __uint_as_float((unsigned)(mykey >> 32));
  float4 bx = make_float4(0.f, 0.f, 0.f, 0.f);
  if (valid) bx = decode_box(loc + ((int64_t)b * P + prior) * 4, priors + (int64_t)prior * 4);
  sbox[tid] = bx;
  __syncthreads();

  // column max of the strictly upper triangular IoU matrix (detection.py:148-150)
  float m = 0.f;
  if (valid) {
    for (int i = 0; i < tid; ++i) m = nan_max(m, box_iou(sbox[i], bx));
  }
  // detection.py:153,160-161: keep = (iou_max <= thresh) [* (scores > conf_thresh)]
  const bool keep = valid && (m <= nms_thresh) && (score > second_thresh);

  int total;
  const int pos = block_excl_scan(keep ? 1 : 0, s_warp, &total);
  if (!CC) {
    const int64_t base = ((int64_t)b * (C - 1) + c) * top_k;
    if (keep) {
      pool_score[base + pos] = score;
      pool_prior[base + pos] = prior;
      reinterpret_cast<float4*>(pool_box)[base + pos] = bx;
    }
    if (tid == 0) pool_n[b * (C - 1) + c] = total;
  } else {
    // cc_fast_nms returns every kept row in descending-score order, no max_dets cut
    // (detection.py:131-133)
    if (keep && pos < max_out) {
      const int64_t o = (int64_t)b * max_out + pos;
      reinterpret_cast<float4*>(out_box)[o] = bx;
      out_score[o] = score;
      out_cls[o] = (int64_t)cand_cls[(int64_t)b * P + prior];
      const float* src = coef + ((int64_t)b * P + prior) * mask_dim;
      for (int k = 0; k < mask_dim; ++k) out_coef[o * mask_dim + k] = src[k];
    }
    cc_zero_rows_from(min(total, max_out));
    if (tid == 0) out_count[b] = min(total, max_out);
  }
}

// ---------------------------------------------------------------------------------------------
// K2 (traditional): per (class, image) greedy NMS -- Detect.traditional_nms (detection.py:182-228)
// with utils/cython_nms.pyx:24-74 as the inner routine.
//   * candidates of class c: score > conf_thresh (detection.py:198); NO top-k cut;
//   * boxes are multiplied by cfg.max_size and areas / intersections use the +1 pixel convention
//     (cython_nms.pyx:31,60-66); box j is suppressed by a kept, higher scoring box i when
//     inter / (area_i + area_j - inter) >= thresh;
//   * the returned box is (box * max_size) / max_size (detection.py:194,228).
// The CTA walks the candidates in descending score order, 256 at a time (exact radix select below
// the previous chunk's smallest key + bitonic sort): each chunk is first tested against the boxes
// kept so far, then resolved sequentially inside the chunk.  Only the first max_keep kept boxes of
// a class can reach the image's top max_keep (they outscore everything later in this class), so
// the walk stops there -- the result is the reference's, without an O(n^2) matrix.
// Ties in score: lower prior index first (the reference's argsort order is unspecified for ties).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float trad_overlap(const float4& a, float area_a, const float4& b, float area_b) {
  const float xx1 = fmaxf(a.x, b.x), yy1 = fmaxf(a.y, b.y);
  const float xx2 = fminf(a.z, b.z), yy2 = fminf(a.w, b.w);
  const float w = fmaxf(0.f, __fadd_rn(__fsub_rn(xx2, xx1), 1.f));
  const float h = fmaxf(0.f, __fadd_rn(__fsub_rn(yy2, yy1), 1.f));
  const float inter = __fmul_rn(w, h);
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
}

__global__ void __launch_bounds__(NT2)
trad_nms_kernel(const float* __restrict__ scoresT, const int32_t* __restrict__ cand_prior,
                const int32_t* __restrict__ cand_count, const float* __restrict__ loc,
                const float* __restrict__ priors, int64_t P, int C, int top_k, float conf_thresh,
                float nms_thresh, float max_size, int max_keep, float* __restrict__ pool_score,
                int32_t* __restrict__ pool_prior, float* __restrict__ pool_box,
                int32_t* __restrict__ pool_n) {
  __shared__ unsigned long long sel[SORT_N];
  __shared__ SelectScratch sc;
  __shared__ float4 sbox[SORT_N];     // current chunk, scaled by max_size
  __shared__ float sarea[SORT_N];
  __shared__ int s_alive[SORT_N];
  __shared__ float4 kbox[SORT_N];     // kept so far (scaled)
  __shared__ float karea[SORT_N];
  __shared__ int s_warp[NT2 / 32];

  const int c = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int M = cand_count[b];
  const float* sc_row = scoresT + ((int64_t)b * (C - 1) + c) * P;
  const int32_t* cp = cand_prior + (int64_t)b * P;
  const int64_t base = ((int64_t)b * (C - 1) + c) * top_k;

  int mine = 0;
  for (int i = tid; i < M; i += NT2) mine += (sc_row[i] > conf_thresh) ? 1 : 0;
  int n_c;
  block_excl_scan(mine, s_warp, &n_c);

  unsigned long long last_key = ~0ull;   // keys of processed candidates are >= last_key
  int kept = 0, processed = 0;
  while (processed < n_c && kept < max_keep) {
    const int K = min(SORT_N, n_c - processed);
    const unsigned long long lk = last_key;
    auto keyfn = [&](int i) -> unsigned long long {
      const float s = sc_row[i];
      if (!(s > conf_thresh)) return 0ull;
      const unsigned long long k =
          ((unsigned long long)__float_as_uint(s) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)cp[i]);
      return k < lk ? k : 0ull;
    };
    block_select_topk(keyfn, M, K, sel, &sc);
    block_sort_desc(sel);

    const unsigned long long mykey = sel[tid];
    const bool valid = tid < K;
    const int prior = valid ? (int)(0xFFFFFFFFu - (unsigned)(mykey & 0xFFFFFFFFull)) : 0;
    const float score = __uint_as_float((unsigned)(mykey >> 32));
    float4 bx = make_float4(0.f, 0.f, 0.f, 0.f);
    float area = 0.f;
    if (valid) {
      const float4 d = decode_box(loc + ((int64_t)b * P + prior) * 4, priors + (int64_t)prior * 4);
      bx = make_float4(__fmul_rn(d.x, max_size), __fmul_rn(d.y, max_size), __fmul_rn(d.z, max_size),
                       __fmul_rn(d.w, max_size));
      area = __fmul_rn(__fadd_rn(__fsub_rn(bx.z, bx.x), 1.f), __fadd_rn(__fsub_rn(bx.w, bx.y), 1.f));
    }
    bool alive = valid;
    for (int k = 0; k < kept && alive; ++k)
      if (trad_overlap(kbox[k], karea[k], bx, area) >= nms_thresh) alive = false;
    sbox[tid] = bx;
    sarea[tid] = area;
    s_alive[tid] = alive ? 1 : 0;
    __syncthreads();
    for (int i = 0; i < K; ++i) {
      if (s_alive[i]) {   // uniform: written before the previous barrier
        if (tid > i && alive && trad_overlap(sbox[i], sarea[i], bx, area) >= nms_thresh) {
          alive = false;
          s_alive[tid] = 0;
        }
      }
      __syncthreads();
    }
    int total;
    const int pos = kept + block_excl_scan(alive ? 1 : 0, s_warp, &total);
    if (alive && pos < max_keep) {
      kbox[pos] = bx;
      karea[pos] = area;
      pool_score[base + pos] = score;
      pool_prior[base + pos] = prior;
      reinterpret_cast<float4*>(pool_box)[base + pos] =
          make_float4(__fdiv_rn(bx.x, max_size), __fdiv_rn(bx.y, max_size), __fdiv_rn(bx.z, max_size),
                      __fdiv_rn(bx.w, max_size));
    }
    kept = min(kept + total, max_keep);
    processed += K;
    last_key = sel[K - 1];
    __syncthreads();   // kbox / sel are rewritten by the next round
  }
  if (tid == 0) pool_n[b * (C - 1) + c] = kept;
}

// ---------------------------------------------------------------------------------------------
// K3: final top max_dets over all (class, rank) pool entries of one image
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT2)
final_select_kernel(const float* __restrict__ pool_score, const int32_t* __restrict__ pool_prior,
                    const float* __restrict__ pool_box, const int32_t* __restrict__ pool_n,
                    const float* __restrict__ coef, int64_t P, int C, int mask_dim, int top_k,
                    int max_dets, int max_out, float* __restrict__ out_box,
                    float* __restrict__ out_coef, int64_t* __restrict__ out_cls,
                    float* __restrict__ out_score, int32_t* __restrict__ out_count) {
  __shared__ unsigned long long sel[SORT_N];
  __shared__ SelectScratch sc;
  __shared__ int s_n[128];  // per-class kept counts (C-1 <= 128)
  __shared__ int s_warp[NT2 / 32];

  const int b = blockIdx.x;
  const int tid = threadIdx.x;
  const int NC = C - 1;
  for (int i = tid; i < NC; i += NT2) s_n[i] = pool_n[b * NC + i];
  __syncthreads();
  int mine = 0;
  for (int i = tid; i < NC; i += NT2) mine += s_n[i];
  int total;
  block_excl_scan(mine, s_warp, &total);
  const int K = min(max_dets, total);
  const float* ps = pool_score + (int64_t)b * NC * top_k;

  auto keyfn = [&](int q) -> unsigned long long {
    int c = q / top_k, r = q - c * top_k;
    if (r >= s_n[c]) return 0ull;
    unsigned hi = __float_as_uint(ps[q]);
    unsigned lo = 0xFFFFFFFFu - (unsigned)q;
    return ((unsigned long long)hi << 32) | (unsigned long long)lo;
  };
  if (K > 0) {
    block_select_topk(keyfn, NC * top_k, K, sel, &sc);
    block_sort_desc(sel);
  }
  __syncthreads();
  if (tid < max_out) {
    const int64_t o = (int64_t)b * max_out + tid;
    if (tid < K) {
      const unsigned long long k = sel[tid];
      const int q = (int)(0xFFFFFFFFu - (unsigned)(k & 0xFFFFFFFFull));
      const int c = q / top_k;
      const int64_t src = (int64_t)b * NC * top_k + q;
      reinterpret_cast<float4*>(out_box)[o] = reinterpret_cast<const float4*>(pool_box)[src];
      out_score[o] = __uint_as_float((unsigned)(k >> 32));
      out_cls[o] = (int64_t)c;
      const float* cs = coef + ((int64_t)b * P + pool_prior[src]) * mask_dim;
      for (int j = 0; j < mask_dim; ++j) out_coef[o * mask_dim + j] = cs[j];
    } else {
      reinterpret_cast<float4*>(out_box)[o] = make_float4(0.f, 0.f, 0.f, 0.f);
      out_score[o] = 0.f;
      out_cls[o] = 0;
      for (int j = 0; j < mask_dim; ++j) out_coef[o * mask_dim + j] = 0.f;
    }
  }
  if (tid == 0) out_count[b] = K;
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

size_t detect_workspace_bytes(int B, int64_t P, int num_classes, int top_k) {
  const size_t NC = (size_t)num_classes - 1;
  size_t s = 0;
  s += align_up((size_t)B * NC * P * sizeof(float), 256);        // scoresT
  s += align_up((size_t)B * P * sizeof(int32_t), 256);           // cand_prior
  s += align_up((size_t)B * P * sizeof(int32_t), 256);           // cand_cls
  s += align_up((size_t)B * sizeof(int32_t), 256);               // cand_count
  s += align_up((size_t)B * NC * top_k * sizeof(float), 256);    // pool_score
  s += align_up((size_t)B * NC * top_k * sizeof(int32_t), 256);  // pool_prior
  s += align_up((size_t)B * NC * top_k * 4 * sizeof(float), 256);  // pool_box
  s += align_up((size_t)B * NC * sizeof(int32_t), 256);          // pool_n
  return s;
}

void detect_workspace_bind(DetectWorkspace* ws, void* base, int B, int64_t P, int num_classes,
                           int top_k) {
  const size_t NC = (size_t)num_classes - 1;
  char* p = (char*)base;
  ws->scoresT = (float*)p;
  p += align_up((size_t)B * NC * P * sizeof(float), 256);
  ws->cand_prior = (int32_t*)p;
  p += align_up((size_t)B * P * sizeof(int32_t), 256);
  ws->cand_cls = (int32_t*)p;
  p += align_up((size_t)B * P * sizeof(int32_t), 256);
  ws->cand_count = (int32_t*)p;
  p += align_up((size_t)B * sizeof(int32_t), 256);
  ws->pool_score = (float*)p;
  p += align_up((size_t)B * NC * top_k * sizeof(float), 256);
  ws->pool_prior = (int32_t*)p;
  p += align_up((size_t)B * NC * top_k * sizeof(int32_t), 256);
  ws->pool_box = (float*)p;
  p += align_up((size_t)B * NC * top_k * 4 * sizeof(float), 256);
  ws->pool_n = (int32_t*)p;
}

void launch_detect(const DetectParams& dp, const float* loc, const float* conf, const float* coef,
                   const float* priors, const DetectWorkspace& ws, float* box, float* coef_out,
                   int64_t* cls, float* score, int32_t* count, cudaStream_t stream,
                   LaunchCounter* lc) {
  YB_REQUIRE(dp.top_k >= 1 && dp.top_k <= SORT_N, "detect: nms_top_k must be in [1,256]");
  YB_REQUIRE(dp.num_classes >= 2 && dp.num_classes - 1 <= 128, "detect: num_classes out of range");
  YB_REQUIRE(dp.max_out <= SORT_N, "detect: max_out must be <= 256");
  YB_REQUIRE(dp.cross_class >= YB_NMS_FAST && dp.cross_class <= YB_NMS_TRADITIONAL, "detect: unknown nms mode");
  YB_REQUIRE(!dp.second_threshold || dp.cross_class == YB_NMS_FAST, "detect: second_threshold exists for fast_nms only");
  YB_REQUIRE(dp.cross_class == YB_NMS_CROSS_CLASS ? dp.max_out >= 1 : dp.max_out >= dp.max_dets,
             "detect: max_out too small");
  YB_REQUIRE(dp.P < (1ll << 31), "detect: too many priors");
  const int B = dp.B, C = dp.num_classes;
  YB_CHECK_CUDA(cudaMemsetAsync(ws.cand_count, 0, sizeof(int32_t) * B, stream));
  {
    dim3 grid((unsigned)ceil_div64(dp.P, K1_ROWS), B);
    const size_t smem = K1_HEADER_BYTES + (size_t)K1_ROWS * C * sizeof(float);
    // past the 48 KB a launch gets by default (C >= 96) the kernel must opt in: 66 KB at C = 129
    if (smem > 48 * 1024)
      YB_CHECK_CUDA(cudaFuncSetAttribute(detect_candidates_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
    detect_candidates_kernel<<<grid, K1_ROWS, smem, stream>>>(
        conf, dp.P, C, dp.conf_is_logits, dp.conf_thresh, dp.cross_class == YB_NMS_CROSS_CLASS ? 1 : 0, ws.scoresT,
        ws.cand_prior,
        ws.cand_cls, ws.cand_count);
    YB_CHECK_LAUNCH();
    if (lc) lc->n++;
  }
  if (dp.cross_class == YB_NMS_CROSS_CLASS) {
    dim3 grid(1, B);
    class_nms_kernel<true><<<grid, NT2, 0, stream>>>(
        ws.scoresT, ws.cand_prior, ws.cand_cls, ws.cand_count, loc, priors, coef, dp.P, C,
        dp.mask_dim, dp.top_k, dp.nms_thresh, -INFINITY, nullptr, nullptr, nullptr, nullptr, dp.max_out, box,
        coef_out, cls, score, count);
    YB_CHECK_LAUNCH();
    if (lc) lc->n++;
  } else {
    dim3 grid(C - 1, B);
    if (dp.cross_class == YB_NMS_TRADITIONAL) {
      YB_REQUIRE(dp.max_dets <= dp.top_k, "detect: traditional NMS needs max_num_detections <= nms_top_k");
      YB_REQUIRE(dp.max_size > 0.f, "detect: traditional NMS needs cfg.max_size");
      trad_nms_kernel<<<grid, NT2, 0, stream>>>(ws.scoresT, ws.cand_prior, ws.cand_count, loc, priors, dp.P, C,
                                                dp.top_k, dp.conf_thresh, dp.nms_thresh, dp.max_size, dp.max_dets,
                                                ws.pool_score, ws.pool_prior, ws.pool_box, ws.pool_n);
    } else {
      class_nms_kernel<false><<<grid, NT2, 0, stream>>>(
          ws.scoresT, ws.cand_prior, ws.cand_cls, ws.cand_count, loc, priors, coef, dp.P, C,
          dp.mask_dim, dp.top_k, dp.nms_thresh, dp.second_threshold ? dp.conf_thresh : -INFINITY, ws.pool_score,
          ws.pool_prior, ws.pool_box, ws.pool_n,
          dp.max_out, nullptr, nullptr, nullptr, nullptr, nullptr);
    }
    YB_CHECK_LAUNCH();
    if (lc) lc->n++;
    final_select_kernel<<<B, NT2, 0, stream>>>(ws.pool_score, ws.pool_prior, ws.pool_box, ws.pool_n,
                                               coef, dp.P, C, dp.mask_dim, dp.top_k, dp.max_dets,
                                               dp.max_out, box, coef_out, cls, score, count);
    YB_CHECK_LAUNCH();
    if (lc) lc->n++;
  }
}

}  // namespace yb
