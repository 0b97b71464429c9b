// Implicit-GEMM convolution on Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
// Replaces cuDNN nn.Conv2d + BatchNorm2d + ReLU (+ residual add) of the reference's backbone /
// FPN / protonet / prediction head (backbone.py:37-57,126-139; yolact.py:311-361,133-212;
// utils/functions.py:163-213) and the SGEMM of DCNv2 (dcn_v2_cuda.cu:149-163).
//
// GEMM view (no im2col buffer anywhere):
//   D[M = output pixels of one spatial tile, N = Cout tile] = sum over taps (r,s) and 64-channel
//   chunks of  A_tap[M, 64] * W_tap[N, 64]^T,   fp16 operands, fp32 accumulation in registers.
// A operand: the activation tensor is NHWC fp16; a 4-D TMA tensor map {C, W, H, B} loads the box
//   {64 channels, tw, th, 1} whose origin is shifted by the tap offset.  Out-of-bounds rows /
//   columns (the conv's zero padding) are zero-filled by TMA itself.  tw*th <= 128 rows land in
//   shared memory as 128-byte rows with the 128B swizzle == the canonical K-major SWIZZLE_128B
//   wgmma layout, so the MMA consumes them with no repacking.
//   Stride-2 convs use one tensor map per input phase (py,px) (a strided *view* of the same
//   buffer: element strides doubled), and the tap table selects (phase map, dx, dy).
// B operand: weights packed [tap][Cout][Cin] fp16, 3-D map, box {64, BN, 1}.
// Pipeline: warpgroup 0 = TMA producer (one thread), warpgroups 1..H = wgmma on their 64-row halves of the tile,
//   then the epilogue from the accumulator registers (+bias -> +residual -> activation -> staged TMA stores).
//   `stages`-deep mbarrier ring (full/empty); each MMA warpgroup frees a slot once its wgmmas have read it.
// CTA pairs (PAIR = true): a cluster of two CTAs computes two adjacent M tiles of the same N tile; each CTA loads
//   its own A tile and HALF of the weight tile, multicast into both CTAs, so the bytes a CTA pulls from L2 per
//   k-block drop from 16 KB + BN*128 to 16 KB + BN*64.  A slot is refilled once the MMA warpgroups of BOTH CTAs
//   have released it.
// Chain kernel (tc_chain_kernel, further down): a run of consecutive layers -- the whole ResNet trunk after the
//   max-pool -- in ONE persistent cooperative launch; the layers' parameter blocks live in global memory, the work
//   units of all layers are dealt round-robin to the CTAs, dependencies are tracked per M tile with counters.
#include <atomic>
#include <vector>
#include "tc_common.cuh"

namespace yb {

using namespace tc;

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;              // fp16 elements = 128 bytes = one swizzle row
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KB
constexpr int MAX_TAPS = 9;
constexpr int MAX_STAGES = 8;

struct alignas(64) TcParams {
  CUtensorMap tmA[4];
  CUtensorMap tmB;
  CUtensorMap tmY;      // output tile store  (epi_tma)
  CUtensorMap tmR;      // residual tile load (epi_tma && residual)
  int epi_tma;          // 1: fp16 NHWC output goes smem -> TMA store, residual comes in by TMA
  int out_off;          // byte offset of the 2 x 16 KB epilogue staging tiles inside dynamic smem
  int res_off;          // byte offset of the residual staging buffers inside dynamic smem
  int m_tiles, n_tiles; // tile = m_tile * n_tiles + n_tile
  int nseg;             // > 0: output channels are split over several fp32 tensors (fused prediction head)
  int seg_begin[3], seg_end[3], seg_ps[3], seg_act[3];
  long long seg_bs[3];
  float* seg_y[3];
  int pdl;              // launched with programmatic stream serialization
  int pair;             // 1: CTA pairs (cluster of 2 sharing the weight tile by multicast)
  int nb;               // batch extent of the tile grid (1 when flattened): tiles with b >= nb are padding
  int ntaps, kchunks, stages;
  int tap_map[MAX_TAPS], tap_dx[MAX_TAPS], tap_dy[MAX_TAPS];
  int tw, th, tiles_x, tiles_y;
  int Ho, Wo, Cout;
  int a_box_bytes;      // tw*th*128
  // epilogue
  void* y;
  const float* bias;
  const __half* residual;
  long long y_batch_stride;
  long long res_batch_stride;
  int y_pix_stride;
  int y_f32;
  int act;
  int vec_ok;
  int res_after_act;
  // split precision (SPLIT kernels): activations are [hi(C) | lo(C)] fp16 pairs per pixel, weights [.. hi(Cin) | lo(Cin)]
  // scaled by a power of two; the accumulator is multiplied by out_scale (its exact inverse) before the bias
  int split;
  int cin;              // logical input channels: the lo plane starts at channel `cin` of the A / B tensor maps
  float out_scale;
  // stream-K (sk != 0): the units' k-block iterations are dealt out in equal contiguous shares, one share per CTA /
  // cluster; a share that ends inside a unit leaves an fp32 partial tile in sk_ws (one slot of 128 x BN floats per
  // CTA) and raises sk_flags[2 * slot]; the CTA holding the unit's FIRST k-blocks adds the partials and runs the
  // epilogue
  int sk;
  float* sk_ws;
  int* sk_flags;
  // split plans with two MMA warpgroups on a flattened (1x1, stride 1) layout read the residual straight from global
  // memory instead of through staging tiles (one more pipeline stage)
  int res_direct;
  int bn;               // N tile (the kernel template's BN; the chain kernel reads it per layer)
};

// ---------------------------------------------------------------------------------------------
// kernel
// ---------------------------------------------------------------------------------------------
// Persistent: CTA c processes tiles c, c + gridDim.x, ...  (tile = m_tile * n_tiles + n_tile).
// Warpgroup 0 is the TMA producer (one thread issues), warpgroups 1..H are the MMA warpgroups: each owns 2/H of the
// tile's two 64-row halves, accumulates them with wgmma in registers and runs the epilogue of its rows.  The producer
// runs up to `stages` k-blocks ahead across tile boundaries, so the loads of tile i+1 overlap the epilogue of tile i.
__device__ __forceinline__ void mma_bar_sync(int nthreads) { asm volatile("bar.sync 1, %0;" ::"r"(nthreads) : "memory"); }

// The k-blocks [k0, k1) of one tile: acc[mh][plane] of 64-row half (cw + mh * H) of the tile (mma_passes; SPLIT: the
// planes are combined into plane 0 at the end).  Each stage is handed back to the producer(s) once the wgmmas that
// read it have completed.
template <int BN, int MH, int H, bool SPLIT, bool PAIR, int NACC>
__device__ __forceinline__ void mma_tile(float (&acc)[MH][SPLIT ? 2 : 1][NACC], uint8_t* smem, uint64_t* full_bar,
                                         uint64_t* empty_bar, int stages, int stage_bytes, int a_bytes, int b_plane_bytes,
                                         uint32_t& kbg, int nkb, int cw, bool signaller) {
  constexpr int NPL = SPLIT ? 2 : 1;
#pragma unroll
  for (int mh = 0; mh < MH; ++mh)
#pragma unroll
    for (int pl = 0; pl < NPL; ++pl)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[mh][pl][i] = 0.f;
  auto release = [&](uint32_t s) {
    if (!signaller) return;
    if (PAIR) {   // the stage's weight half of EACH CTA is refilled by both producers: free it in both
      mbar_arrive_cluster(mapa_u32(smem_u32(&empty_bar[s]), 0));
      mbar_arrive_cluster(mapa_u32(smem_u32(&empty_bar[s]), 1));
    } else {
      mbar_arrive(&empty_bar[s]);
    }
  };
  for (int kb = 0; kb < nkb; ++kb, ++kbg) {
    const uint32_t s = kbg % (uint32_t)stages;
    mbar_wait(&full_bar[s], (kbg / (uint32_t)stages) & 1u);
    const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes);
    const uint32_t sb = sa + (uint32_t)a_bytes;
    wgmma_fence();
#pragma unroll
    for (int mh = 0; mh < MH; ++mh) {
      const uint32_t half_off = (uint32_t)(cw + mh * H) * (64u * 128u);
      mma_passes<BN, BLOCK_K / 16, SPLIT>(
          acc[mh][0], acc[mh][NPL - 1],
          [&](int pl, int k) { return make_sw128_desc(sa + (uint32_t)(pl * A_STAGE_BYTES) + half_off) + (uint64_t)(2 * k); },
          [&](int pl, int k) { return make_sw128_desc(sb + (uint32_t)(pl * b_plane_bytes)) + (uint64_t)(2 * k); });
    }
    wgmma_commit();
    if (stages == 1) {   // a single stage: the next k-block can only land once these wgmmas have read this one
      wgmma_wait<0>();
      release(s);
    } else if (kb > 0) {   // the previous k-block's wgmmas are done: its stage can be refilled
      wgmma_wait<1>();
      release((kbg - 1) % (uint32_t)stages);
    }
  }
  wgmma_wait<0>();
  if (nkb > 0 && stages > 1) release((kbg - 1) % (uint32_t)stages);
#pragma unroll
  for (int mh = 0; mh < MH; ++mh)
#pragma unroll
    for (int pl = 0; pl < NPL; ++pl) fence_regs<BN / 2>(acc[mh][pl]);
  if (SPLIT) {
#pragma unroll
    for (int mh = 0; mh < MH; ++mh)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[mh][0][i] = split_combine(acc[mh][0][i], acc[mh][NPL - 1][i]);
  }
}

// Staged epilogue of the 64-channel chunks [0, nchunks) of a tile: (* out_scale) + bias, + residual (a swizzled smem
// tile loaded by TMA, or -- res_g, flattened layouts -- straight from global memory), activation, fp16 pack into the
// swizzled 128-row staging tile, one TMA store per chunk (and plane) by thread 0 of the MMA warpgroups (OOB rows are
// clipped by the tensor map).  SPLIT: the result is written as hi / lo = rn(v - hi) into two staging tiles.
// g: chunks staged by this CTA so far (buffer = g % NBUF).  has_res_tile: res_tmap holds the residual; the load of the
// tile's chunk 0 was issued before its main loop, chunk c + 1 is requested here.
struct EpiArgs {
  const CUtensorMap* tmY;
  const CUtensorMap* tmR;
  uint64_t* res_full_bar;
  uint8_t* out_base;
  uint8_t* res_base;
  const float* bias;
  const __half* res_g;   // res_direct: residual of pixel (x0 + row), channel n0, hi plane (lo plane Cout halfs further)
  int res_pix_stride;    // halfs per residual pixel (both planes)
  uint32_t res_tx;       // bytes of one residual chunk (all planes): the box holds tw*th rows, not always 128
  int Wo, Cout, n0, x0, y0, b, nchunks, nbuf;
  float out_scale;
};
template <int ACT, bool RES_AFTER, bool SPLIT, int BN, int MH, int H, int NACC>
__device__ __forceinline__ void epi_staged(float (&acc)[MH][SPLIT ? 2 : 1][NACC], const EpiArgs& e, bool has_res_tile,
                                           uint32_t& g, int cw, int ct, int lane, int wq) {
  constexpr int NPL = SPLIT ? 2 : 1;
  const int nthreads = 128 * H;
#pragma unroll
  for (int c = 0; c < BN / 64; ++c) {
    if (c >= e.nchunks) break;
    const uint32_t buf = (e.nbuf == 1) ? 0u : (g & 1u);
    uint8_t* out_tile = e.out_base + buf * (NPL * A_STAGE_BYTES);
    const uint8_t* res_tile = e.res_base + buf * (NPL * A_STAGE_BYTES);
    if (g >= (uint32_t)e.nbuf) {
      if (ct == 0) {
        if (e.nbuf == 1) bulk_wait_read<0>(); else bulk_wait_read<1>();   // the store that last used this tile has read it
      }
      mma_bar_sync(nthreads);
    }
    if (has_res_tile) {
      if (ct == 0 && e.nbuf == 2 && c + 1 < e.nchunks) {   // next chunk's residual into the other buffer
        const uint32_t nb = (g + 1) & 1u;
        mbar_expect_tx(&e.res_full_bar[nb], e.res_tx);
#pragma unroll
        for (int pl = 0; pl < NPL; ++pl)
          tma_load_4d(e.res_base + nb * (NPL * A_STAGE_BYTES) + pl * A_STAGE_BYTES, e.tmR, &e.res_full_bar[nb],
                      e.n0 + (c + 1) * 64 + pl * e.Cout, e.x0, e.y0, e.b);
      }
      mbar_wait(&e.res_full_bar[buf], (e.nbuf == 1) ? (g & 1u) : ((g >> 1) & 1u));
    }
    const int nbase = e.n0 + c * 64;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = 8 * j + 2 * (lane & 3);
      const float b0 = (e.bias && nbase + col < e.Cout) ? __ldg(e.bias + nbase + col) : 0.f;
      const float b1 = (e.bias && nbase + col + 1 < e.Cout) ? __ldg(e.bias + nbase + col + 1) : 0.f;
#pragma unroll
      for (int mh = 0; mh < MH; ++mh)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = (cw + mh * H) * 64 + wq * 16 + (lane >> 2) + 8 * h;
          const int i = (c * 8 + j) * 4 + 2 * h;
          float v0 = scale_bias<SPLIT>(acc[mh][0][i], e.out_scale, b0);
          float v1 = scale_bias<SPLIT>(acc[mh][0][i + 1], e.out_scale, b1);
          if (RES_AFTER) {
            v0 = act_t<ACT>(v0);
            v1 = act_t<ACT>(v1);
          }
          const uint32_t off = sw128_off((uint32_t)row, (uint32_t)j) + (uint32_t)(lane & 3) * 4u;
          if (has_res_tile || e.res_g) {
            __half2 rh, rl;
            if (has_res_tile) {
              rh = *reinterpret_cast<const __half2*>(res_tile + off);
              if (SPLIT) rl = *reinterpret_cast<const __half2*>(res_tile + A_STAGE_BYTES + off);
            } else if (e.x0 + row < e.Wo) {   // L2: inside a chain other SMs wrote it during this launch
              const __half* rp = e.res_g + (size_t)row * e.res_pix_stride + c * 64 + col;
              const unsigned int u = __ldcg(reinterpret_cast<const unsigned int*>(rp));
              rh = *reinterpret_cast<const __half2*>(&u);
              if (SPLIT) {
                const unsigned int ul = __ldcg(reinterpret_cast<const unsigned int*>(rp + e.Cout));
                rl = *reinterpret_cast<const __half2*>(&ul);
              }
            } else {
              rh = rl = __floats2half2_rn(0.f, 0.f);
            }
            // one plane at a time, (v + hi) + lo: v + split2_to_f32(rh, rl) rounds differently
            const float2 f = __half22float2(rh);
            v0 += f.x;
            v1 += f.y;
            if (SPLIT) {
              const float2 fl = lo2_to_f32(rl);
              v0 += fl.x;
              v1 += fl.y;
            }
          }
          if (!RES_AFTER) {
            v0 = act_t<ACT>(v0);
            v1 = act_t<ACT>(v1);
          }
          __half2 hi, lo;
          if (SPLIT) split2_from_f32(v0, v1, hi, lo);
          else hi = f16x2_from_f32(v0, v1);
          *reinterpret_cast<__half2*>(out_tile + off) = hi;
          if (SPLIT) *reinterpret_cast<__half2*>(out_tile + A_STAGE_BYTES + off) = lo;
        }
    }
    fence_proxy_async();   // generic-proxy smem writes -> visible to the TMA (async proxy)
    mma_bar_sync(nthreads);
    if (ct == 0) {
      tma_store_4d(e.tmY, out_tile, nbase, e.x0, e.y0, e.b);
      if (SPLIT) tma_store_4d(e.tmY, out_tile + A_STAGE_BYTES, nbase + e.Cout, e.x0, e.y0, e.b);
      bulk_commit();
      if (has_res_tile && e.nbuf == 1 && c + 1 < e.nchunks) {   // single buffer: refill it now that it has been read
        mbar_expect_tx(&e.res_full_bar[0], e.res_tx);
#pragma unroll
        for (int pl = 0; pl < NPL; ++pl)
          tma_load_4d(e.res_base + pl * A_STAGE_BYTES, e.tmR, &e.res_full_bar[0], e.n0 + (c + 1) * 64 + pl * e.Cout, e.x0,
                      e.y0, e.b);
      }
    }
    ++g;
  }
}

template <bool SPLIT, int BN, int MH, int H, int NACC>
__device__ __forceinline__ void epi_staged_act(int act, int raa, float (&acc)[MH][SPLIT ? 2 : 1][NACC], const EpiArgs& e,
                                               bool has_res_tile, uint32_t& g, int cw, int ct, int lane, int wq) {
  switch (act) {
    case ACT_RELU: epi_staged<ACT_RELU, false, SPLIT, BN, MH, H>(acc, e, has_res_tile, g, cw, ct, lane, wq); break;
    case ACT_LEAKY:
      if (raa) epi_staged<ACT_LEAKY, true, SPLIT, BN, MH, H>(acc, e, has_res_tile, g, cw, ct, lane, wq);
      else epi_staged<ACT_LEAKY, false, SPLIT, BN, MH, H>(acc, e, has_res_tile, g, cw, ct, lane, wq);
      break;
    case ACT_TANH: epi_staged<ACT_TANH, false, SPLIT, BN, MH, H>(acc, e, has_res_tile, g, cw, ct, lane, wq); break;
    default: epi_staged<ACT_NONE, false, SPLIT, BN, MH, H>(acc, e, has_res_tile, g, cw, ct, lane, wq); break;
  }
}

struct TileCoord {
  int b, x0, y0, n0;
};
__device__ __forceinline__ TileCoord decode_mn(const TcParams& p, int m, int nt, int BN) {
  TileCoord t;
  const int tx = m % p.tiles_x;
  m /= p.tiles_x;
  const int ty = m % p.tiles_y;
  t.b = m / p.tiles_y;
  t.x0 = tx * p.tw;
  t.y0 = ty * p.th;
  t.n0 = nt * BN;
  return t;
}
// Work unit u of a CTA: one (M tile, N tile).  Single CTAs walk tiles; a CTA pair walks (M-tile pair, N tile)
// units, CTA `rank` taking M tile 2*group + rank (a padding tile when the M-tile count is odd: its loads are
// zero-filled and its stores clipped by the tensor maps, b >= nb marks it for the direct epilogue).
template <bool PAIR>
__device__ __forceinline__ TileCoord decode_unit(const TcParams& p, int u, int rank, int BN) {
  const int nt = u % p.n_tiles;
  const int mg = u / p.n_tiles;
  return decode_mn(p, PAIR ? 2 * mg + rank : mg, nt, BN);
}

// Work of one CTA (cluster): a list of segments (unit, [k0, k1)).  Without stream-K: whole units unit0, unit0 + step, ...
// With stream-K: the contiguous iteration range [cid * I / G, (cid + 1) * I / G) of I = units * k-blocks, cut at unit
// boundaries -- so a CTA's first segment may be the TAIL of a unit (k0 > 0: dumped as a partial) and its last one the
// HEAD of a unit (k0 == 0, k1 < num_kb: this CTA collects the partials and finishes the unit).
struct WorkIter {
  int num_kb, num_units, ustep, sk, u;
  long long it, it_hi;
  __device__ __forceinline__ static long long share_lo(long long total, int c, int G) { return total * c / G; }
  __device__ __forceinline__ void init(int sk_, int num_kb_, int num_units_, int unit0, int ustep_) {
    sk = sk_;
    num_kb = num_kb_;
    num_units = num_units_;
    ustep = ustep_;
    u = unit0;
    const long long total = (long long)num_units_ * num_kb_;
    it = share_lo(total, unit0, ustep_);
    it_hi = share_lo(total, unit0 + 1, ustep_);
  }
  __device__ __forceinline__ bool next(int& uu, int& k0, int& k1) {
    if (!sk) {
      if (u >= num_units) return false;
      uu = u;
      k0 = 0;
      k1 = num_kb;
      u += ustep;
      return true;
    }
    if (it >= it_hi) return false;
    uu = (int)(it / num_kb);
    k0 = (int)(it - (long long)uu * num_kb);
    const long long rem = it_hi - it;
    k1 = (rem < (long long)(num_kb - k0)) ? (int)(k0 + rem) : num_kb;
    it += k1 - k0;
    return true;
  }
};

template <int BN, bool PAIR, int H, bool SPLIT>
__global__ void __launch_bounds__(128 * (1 + H), 1)
tc_conv_kernel(const __grid_constant__ TcParams p) {
  // SPLIT (YB_PREC_F16X3): every operand has a hi and a (2^11-scaled) lo fp16 plane; a k-block stages A_hi, A_lo, W_hi,
  // W_lo (see mma_tile).
  constexpr int NPL = SPLIT ? 2 : 1;
  constexpr int MH = 2 / H;
  constexpr int NACC = BN / 2;
  static_assert(MH * NPL * NACC <= 128, "accumulator tile exceeds the register budget");
  constexpr int B_PLANE_BYTES = BN * BLOCK_K * 2;   // a pair CTA loads half of it and receives the peer's half
  constexpr int A_BYTES = NPL * A_STAGE_BYTES;
  constexpr int STAGE_BYTES = A_BYTES + NPL * B_PLANE_BYTES;

  extern __shared__ uint8_t smem_dyn[];
  __shared__ uint64_t full_bar[MAX_STAGES];
  __shared__ uint64_t empty_bar[MAX_STAGES];
  __shared__ uint64_t res_full_bar[2];

  // 1024-byte alignment required by SWIZZLE_128B (host adds 1024 bytes of slack)
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int stages = p.stages;
  const int num_kb = p.ntaps * p.kchunks;
  const int rank = PAIR ? (int)cluster_ctarank() : 0;
  const int unit0 = PAIR ? (int)cluster_id_x() : (int)blockIdx.x;
  const int ustep = PAIR ? (int)cluster_nclusters_x() : (int)gridDim.x;
  const int num_units = (PAIR ? (p.m_tiles + 1) / 2 : p.m_tiles) * p.n_tiles;

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], (PAIR ? 2 : 1) * H);   // one arrival per MMA warpgroup (of both CTAs of a pair)
    }
    for (int i = 0; i < 2; ++i) mbar_init(&res_full_bar[i], 1);
    fence_barrier_init();
    tma_prefetch_desc(&p.tmB);
    tma_prefetch_desc(&p.tmA[0]);
    if (p.epi_tma) tma_prefetch_desc(&p.tmY);
  }
  __syncthreads();
  if (PAIR) cluster_sync_all();   // the peer's barriers are initialised before anything signals them
  // Programmatic dependent launch: everything above overlaps the tail of the previous kernel in the stream, and so do
  // the WEIGHT tiles of this CTA's first k-blocks (constants: they do not depend on the previous layer); the
  // activations are only touched after griddepcontrol.wait.  Dependents are released at once: they can become resident
  // (and do the same) as soon as an SM has room -- which needs a plan that leaves room (plan->pdl_friendly).
  uint32_t pre = 0;   // producer thread only: k-blocks whose weight tile is already in flight
  if (p.pdl) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (!PAIR && !SPLIT && !p.sk && threadIdx.x == 0 && unit0 < num_units) {   // (a stream-K walk starts mid-unit)
      const TileCoord t0 = decode_unit<PAIR>(p, unit0, rank, BN);
      const int npre = min(stages, num_kb);
      for (int kb = 0; kb < npre; ++kb) {
        const int tap = kb / p.kchunks;
        const int kc = kb - tap * p.kchunks;
        mbar_expect_tx(&full_bar[kb], (uint32_t)p.a_box_bytes + (uint32_t)B_PLANE_BYTES);
        tma_load_3d(smem + (size_t)kb * STAGE_BYTES + A_BYTES, &p.tmB, &full_bar[kb], kc * BLOCK_K, t0.n0, tap);
      }
      pre = (uint32_t)npre;
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");
  }

  if (warp < 4) {
    // ===================== TMA producer warpgroup (one thread issues) =====================
    if (threadIdx.x == 0) {
      const uint32_t tx_bytes = ((uint32_t)p.a_box_bytes + (uint32_t)B_PLANE_BYTES) * (uint32_t)NPL;
      uint32_t kbg = 0;
      WorkIter wi;
      wi.init(p.sk, num_kb, num_units, unit0, ustep);
      int u, k0, k1;
      while (wi.next(u, k0, k1)) {
        const TileCoord tc_ = decode_unit<PAIR>(p, u, rank, BN);
        for (int kb = k0; kb < k1; ++kb, ++kbg) {
          const uint32_t s = kbg % (uint32_t)stages;
          const uint32_t it = kbg / (uint32_t)stages;
          mbar_wait(&empty_bar[s], (it & 1u) ^ 1u);
          const int tap = kb / p.kchunks;
          const int kc = kb - tap * p.kchunks;
          uint8_t* sa = smem + (size_t)s * STAGE_BYTES;
          uint8_t* sb = sa + A_BYTES;
          const CUtensorMap* ma = &p.tmA[p.tap_map[tap]];
          const int ax = tc_.x0 + p.tap_dx[tap], ay = tc_.y0 + p.tap_dy[tap];
          if (PAIR) {
            // own A tile; own half of the weight tile, multicast into both CTAs (each barrier expects both halves)
            mbar_expect_tx(&full_bar[s], tx_bytes);
#pragma unroll
            for (int pl = 0; pl < NPL; ++pl) {
              tma_load_4d(sa + pl * A_STAGE_BYTES, ma, &full_bar[s], kc * BLOCK_K + pl * p.cin, ax, ay, tc_.b);
              tma_load_3d_mc(sb + pl * B_PLANE_BYTES + rank * (B_PLANE_BYTES / 2), &p.tmB, &full_bar[s], (uint16_t)3,
                             kc * BLOCK_K + pl * p.cin, tc_.n0 + rank * (BN / 2), tap);
            }
          } else if (!SPLIT && kbg < pre) {
            // PDL: this stage was armed and its weight tile requested before the dependency wait
            tma_load_4d(sa, ma, &full_bar[s], kc * BLOCK_K, ax, ay, tc_.b);
          } else {
            mbar_expect_tx(&full_bar[s], tx_bytes);
#pragma unroll
            for (int pl = 0; pl < NPL; ++pl) {
              tma_load_4d(sa + pl * A_STAGE_BYTES, ma, &full_bar[s], kc * BLOCK_K + pl * p.cin, ax, ay, tc_.b);
              tma_load_3d(sb + pl * B_PLANE_BYTES, &p.tmB, &full_bar[s], kc * BLOCK_K + pl * p.cin, tc_.n0, tap);
            }
          }
        }
      }
    }
  } else {
    // ===================== MMA warpgroups: main loop + epilogue =====================
    const int cw = warp / 4 - 1;              // MMA warpgroup
    const int ct = threadIdx.x - 128;         // 0 .. 128*H - 1
    const int wq = warp & 3;
    const bool signaller = (threadIdx.x & 127) == 0;
    const bool has_res_tile = (p.residual != nullptr) && !p.res_direct && p.epi_tma;
    const int nbuf = SPLIT ? 1 : 2;            // staging / residual buffers (a buffer = NPL tiles of 16 KB)
    uint8_t* out_base = smem + p.out_off;
    uint8_t* res_base = smem + p.res_off;
    float acc[MH][NPL][NACC];
    uint32_t kbg = 0, g = 0;
    WorkIter wi;
    wi.init(p.sk, num_kb, num_units, unit0, ustep);
    int u, k0, k1;
    // stream-K bookkeeping: this CTA's workspace slot, and (for the head of a split unit) the slots it collects
    const int sk_slot = PAIR ? 2 * unit0 + rank : unit0;
    while (wi.next(u, k0, k1)) {
      const TileCoord tc_ = decode_unit<PAIR>(p, u, rank, BN);
      const bool sk_dump = (k0 > 0);                       // tail / middle of a unit: leave a partial tile
      const bool sk_head = (k0 == 0 && k1 < num_kb);       // head of a split unit: add the partials, then finish
      const int x0 = tc_.x0, y0 = tc_.y0, b = tc_.b, n0 = tc_.n0;
      const int nchunks = (min(BN, p.Cout - n0) + 63) >> 6;
      if (has_res_tile && !sk_dump && ct == 0) {   // the residual of chunk 0 travels during the main loop
        const uint32_t buf = (nbuf == 1) ? 0u : (g & 1u);
        mbar_expect_tx(&res_full_bar[buf], (uint32_t)p.a_box_bytes * (uint32_t)NPL);
#pragma unroll
        for (int pl = 0; pl < NPL; ++pl)
          tma_load_4d(res_base + buf * (NPL * A_STAGE_BYTES) + pl * A_STAGE_BYTES, &p.tmR, &res_full_bar[buf],
                      n0 + pl * p.Cout, x0, y0, b);
      }
      mma_tile<BN, MH, H, SPLIT, PAIR>(acc, smem, full_bar, empty_bar, stages, STAGE_BYTES, A_BYTES, B_PLANE_BYTES, kbg,
                                       k1 - k0, cw, signaller);
      // stream-K partial tiles: slot-major, then accumulator register, then thread (coalesced)
      const size_t ws_stride = (size_t)128 * H;
      if (sk_dump) {
        float* w = p.sk_ws + (size_t)sk_slot * BLOCK_M * BN + ct;
#pragma unroll
        for (int mh = 0; mh < MH; ++mh)
#pragma unroll
          for (int i = 0; i < NACC; ++i) __stcg(w + (mh * NACC + i) * ws_stride, acc[mh][0][i]);
        __threadfence();     // the partial is visible device-wide before the flag
        mma_bar_sync(128 * H);
        if (ct == 0) st_release_gpu(p.sk_flags + 2 * sk_slot, 1);
        continue;
      }
      int sk_parts = 0;
      if (sk_head) {   // the partial tiles of this unit's other k ranges (the following CTAs / clusters left them first thing)
        const long long total = (long long)num_units * num_kb, unit_end = (long long)(u + 1) * num_kb;
        while (unit0 + 1 + sk_parts < ustep && WorkIter::share_lo(total, unit0 + 1 + sk_parts, ustep) < unit_end) ++sk_parts;
        if (ct == 0)
          for (int j = 1; j <= sk_parts; ++j) {
            const int* f = p.sk_flags + 2 * (PAIR ? 2 * (unit0 + j) + rank : unit0 + j);
            while (ld_acquire_gpu(f) == 0) {
            }
          }
        mma_bar_sync(128 * H);
        for (int j = 1; j <= sk_parts; ++j) {
          const int slot = PAIR ? 2 * (unit0 + j) + rank : unit0 + j;
          const float* w = p.sk_ws + (size_t)slot * BLOCK_M * BN + ct;
#pragma unroll
          for (int mh = 0; mh < MH; ++mh)
#pragma unroll
            for (int i = 0; i < NACC; ++i) acc[mh][0][i] += __ldcg(w + (mh * NACC + i) * ws_stride);
        }
      }
      if (p.epi_tma) {
        EpiArgs e;
        e.tmY = &p.tmY;
        e.tmR = &p.tmR;
        e.res_full_bar = res_full_bar;
        e.out_base = out_base;
        e.res_base = res_base;
        e.bias = p.bias;
        // res_direct (flattened 1x1 layouts only): pixel = x0 + row, both planes of the pixel are contiguous
        e.res_g = (p.res_direct && p.residual) ? p.residual + (size_t)x0 * (size_t)(NPL * p.Cout) + n0 : nullptr;
        e.res_pix_stride = NPL * p.Cout;
        e.res_tx = (uint32_t)p.a_box_bytes * (uint32_t)NPL;
        e.Wo = p.Wo;
        e.Cout = p.Cout;
        e.n0 = n0;
        e.x0 = x0;
        e.y0 = y0;
        e.b = b;
        e.nchunks = nchunks;
        e.nbuf = nbuf;
        e.out_scale = p.out_scale;
        epi_staged_act<SPLIT, BN, MH, H>(p.act, p.res_after_act, acc, e, has_res_tile, g, cw, ct, lane, wq);
      } else {
        // ---- direct epilogue (fp32 / unaligned outputs: the head tensors): each thread stores its fragment's
        //      channel pairs of its rows
        const int ncols = min(BN, p.Cout - n0);
        const int raa = p.res_after_act;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          if (8 * j >= ncols) break;
#pragma unroll
          for (int e2 = 0; e2 < 2; ++e2) {
            const int cl = 8 * j + 2 * (lane & 3) + e2;
            if (cl >= ncols) continue;
            const int n = n0 + cl;
            const float bias_n = p.bias ? __ldg(p.bias + n) : 0.f;
            int act = p.act;
            // fused prediction head: this channel belongs to one of up to 3 output tensors
            float* seg_base = nullptr;
            long long seg_bs = 0;
            int seg_ps = 0, seg_c = 0;
            if (p.nseg > 0) {
#pragma unroll
              for (int sg = 0; sg < 3; ++sg)
                if (sg < p.nseg && n >= p.seg_begin[sg] && n < p.seg_end[sg]) {
                  seg_base = p.seg_y[sg];
                  seg_bs = p.seg_bs[sg];
                  seg_ps = p.seg_ps[sg];
                  seg_c = n - p.seg_begin[sg];
                  act = p.seg_act[sg];
                }
            }
#pragma unroll
            for (int mh = 0; mh < MH; ++mh)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int trow = (cw + mh * H) * 64 + wq * 16 + (lane >> 2) + 8 * h;
                const int ty_ = trow / p.tw, tx_ = trow - ty_ * p.tw;
                const int oy = y0 + ty_, ox = x0 + tx_;
                if (trow >= p.tw * p.th || oy >= p.Ho || ox >= p.Wo || b >= p.nb) continue;
                const long long pix = (long long)oy * p.Wo + ox;
                const float a = acc[mh][0][j * 4 + 2 * h + e2];
                float v = scale_bias<SPLIT>(a, p.out_scale, bias_n);
                float rsd = 0.f;
                if (p.residual) {
                  const __half* rp = p.residual + ((long long)b * p.res_batch_stride + pix * p.Cout) * NPL + n;
                  rsd = SPLIT ? split_to_f32(rp[0], rp[p.Cout]) : __half2float(rp[0]);
                }
                if (!raa) v += rsd;
                v = apply_act(v, act);
                if (raa) v += rsd;
                if (p.nseg > 0) {
                  if (seg_base) seg_base[(long long)b * seg_bs + pix * seg_ps + seg_c] = v;
                  continue;
                }
                const long long o = (long long)b * p.y_batch_stride + pix * p.y_pix_stride + n;
                if (p.y_f32) {
                  reinterpret_cast<float*>(p.y)[o] = v;
                } else if (SPLIT) {   // y_pix_stride counts halfs and already includes both planes
                  __half hi, lo;
                  split_f32(v, hi, lo);
                  reinterpret_cast<__half*>(p.y)[o] = hi;
                  reinterpret_cast<__half*>(p.y)[o + p.Cout] = lo;
                } else {
                  reinterpret_cast<__half*>(p.y)[o] = from_f32<__half>(v);
                }
              }
          }
        }
      }
      if (sk_head) {   // every thread has read the partials: re-arm the flags
        mma_bar_sync(128 * H);
        if (ct == 0)
          for (int j = 1; j <= sk_parts; ++j) st_relaxed_gpu(p.sk_flags + 2 * (PAIR ? 2 * (unit0 + j) + rank : unit0 + j), 0);
      }
    }
    if (p.epi_tma && ct == 0) bulk_wait_read<0>();  // smem must outlive the bulk reads
  }

  __syncthreads();
  if (PAIR) cluster_sync_all();   // no CTA leaves while its peer may still multicast into it or signal its barriers
}

// ---------------------------------------------------------------------------------------------
// chain kernel: a run of consecutive convolutions (the 1x1 -> 3x3 -> 1x1 (+residual) bottleneck blocks of one ResNet
// stage, backbone.py:37-57) in ONE persistent launch
// ---------------------------------------------------------------------------------------------
// Every layer of the chain is an ordinary plan of the shape <BN = 128 or 64, single CTA, two MMA warpgroups,
// staged TMA epilogue, residual read from global memory>; their parameter blocks (tensor maps included) sit in an array in global
// memory.  The work units of all layers form ONE list (layer-major, then M tile, then N tile) that is dealt round-robin
// to the CTAs (one per SM), so a CTA moves from its last tile of layer L straight to its first tile of layer L + 1: no launch,
// no prologue (barriers, descriptor fetch), no tail where most SMs idle -- the TMA ring and the
// staging tiles of a CTA simply keep running across the layer boundary.
// Dependencies are tracked per M tile instead of by a grid-wide barrier: thread 0 of the MMA warpgroups bumps done[layer][m tile]
// once the stores of a tile have completed; before the first ACTIVATION load of a tile the producer warp waits until
// every tile of the layer that produces its input which overlaps the input rows the tile reads (its own rows mapped
// through stride / padding / kernel height), and every tile of the layer that produces its residual which overlaps its
// own rows, has been finished by all its N tiles (the weight tiles of the first k-blocks are requested before the
// wait).  Layers may differ in resolution (stride-2 layers), N tile (64 / 128) and tile shape.  All dependencies point
// backwards in the unit list and every CTA walks its units in list order, so the earliest unfinished unit can always
// run: no deadlock as long as the CTAs are co-resident (cooperative launch, one CTA per SM).
// Every activation has its own buffer (engine.cu alloc_act: nothing is recycled inside a forward pass), so there are
// no write-after-read hazards to order.
struct ChainLayer {
  int ubase;               // position of this layer's unit 0 in the chain's unit list
  int units;               // m_tiles * n_tiles
  int flat;                // 1: tile m = pixels [m * tw, m * tw + tw) of the flattened B*H*W axis; 0: tiles_x x tiles_y tiles per image
  int W, H, rows;          // OUTPUT image size; rows = B * H  (global row r = b * H + y, pixel = r * W + x)
  int tw, th, tiles_x, tiles_y;
  int done_off;            // this layer's counters: done[done_off + m_tile]
  int target;              // a finished M tile: n_tiles (each N tile adds 1 once its stores have completed)
  int dep_a;               // chain layer that writes this layer's input (-1: a tensor complete before the launch)
  int dep_r;               // chain layer that writes this layer's residual (-1: none / outside / implied by dep_a's own dependencies)
  int stride, pad, kh;     // output row y reads input rows [y * stride - pad, y * stride - pad + kh)
};

// The dependency arithmetic, shared by the kernel and a host mirror (yb_debug_chain_deps: CPU property tests).
// Global output rows [r0, r1] of M tile m of layer ci
__host__ __device__ __forceinline__ void chain_rows_of_tile(const ChainLayer& ci, int m, int& r0, int& r1) {
  if (ci.flat) {
    const int lo = m * ci.tw;
    int hi = lo + ci.tw;
    if (hi > ci.rows * ci.W) hi = ci.rows * ci.W;
    r0 = lo / ci.W;
    r1 = (hi - 1) / ci.W;
  } else {
    const int ty = (m / ci.tiles_x) % ci.tiles_y, b = m / (ci.tiles_x * ci.tiles_y);
    int y1 = ty * ci.th + ci.th;
    if (y1 > ci.H) y1 = ci.H;
    r0 = b * ci.H + ty * ci.th;
    r1 = b * ci.H + y1 - 1;
  }
}
// Rows [ra, rb] of the input tensor (written by layer pa: its image height differs under a stride) that output rows
// [r0, r1] of layer ci read
__host__ __device__ __forceinline__ void chain_input_rows(const ChainLayer& ci, const ChainLayer& pa, int r0, int r1, int& ra, int& rb) {
  const int b0 = r0 / ci.H, y0 = r0 - b0 * ci.H, b1 = r1 / ci.H, y1 = r1 - b1 * ci.H;
  int lo = y0 * ci.stride - ci.pad, hi = y1 * ci.stride - ci.pad + ci.kh - 1;
  if (lo < 0) lo = 0;
  if (hi > pa.H - 1) hi = pa.H - 1;
  ra = b0 * pa.H + lo;
  rb = b1 * pa.H + hi;
}
// M tiles of layer `pi` that overlap its global rows [ra, rb]
__host__ __device__ __forceinline__ void chain_tiles_of_rows(const ChainLayer& pi, int ra, int rb, int& ia, int& ib) {
  if (pi.flat) {
    ia = (ra * pi.W) / pi.tw;
    ib = ((rb + 1) * pi.W - 1) / pi.tw;
  } else {
    const int ba = ra / pi.H, ya = ra - ba * pi.H, bb = rb / pi.H, yb = rb - bb * pi.H;
    ia = (ba * pi.tiles_y + ya / pi.th) * pi.tiles_x;
    ib = (bb * pi.tiles_y + yb / pi.th) * pi.tiles_x + pi.tiles_x - 1;
  }
}

// pipeline stages of the chain kernel: the ring plus NPL x 16 KB staging tiles per buffer (two buffers in the fp16 mode,
// one in the split mode) fill the 227 KB of an SM
__host__ __device__ constexpr int chain_stages(bool split) { return split ? 3 : 6; }

// first unit of a layer that belongs to CTA `cta` when the chain's unit list is dealt round-robin over G CTAs
__device__ __forceinline__ int chain_first_unit(int cta, int ubase, int G) {
  int r = (cta - ubase) % G;
  return r < 0 ? r + G : r;
}

template <bool SPLIT>
__global__ void __launch_bounds__(384, 1)
tc_chain_kernel(const TcParams* __restrict__ layers, const ChainLayer* __restrict__ info, int nl, int* __restrict__ done,
                long long* __restrict__ stats) {
  // stats (diagnostics, YB_CHAIN_STATS=1; null otherwise): per CTA 8 counters of SM cycles spent waiting --
  // [0] producer: dependency counters, [1] producer: free ring slot, [4] MMA warpgroups: store completion before a
  // signal, [6] whole kernel (the others stay 0)
  const long long t_kernel0 = stats ? clock64() : 0;
  long long w0 = 0, w1 = 0;
  constexpr int NPL = SPLIT ? 2 : 1;
  constexpr int B_PLANE_BYTES = 128 * BLOCK_K * 2;
  constexpr int A_BYTES = NPL * A_STAGE_BYTES;
  constexpr int STAGE_BYTES = A_BYTES + NPL * B_PLANE_BYTES;
  constexpr int stages = chain_stages(SPLIT);

  extern __shared__ uint8_t smem_dyn[];
  __shared__ uint64_t full_bar[MAX_STAGES];
  __shared__ uint64_t empty_bar[MAX_STAGES];

  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  uint8_t* out_base = smem + stages * STAGE_BYTES;
  const int G = (int)gridDim.x;
  const int cta = (int)blockIdx.x;

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);
    }
    fence_barrier_init();
    tma_prefetch_desc(&layers[0].tmB);
    tma_prefetch_desc(&layers[0].tmA[0]);
    tma_prefetch_desc(&layers[0].tmY);
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer (lane 0 of warp 0 issues; warp 0 polls the dependency counters) =====================
    if (warp == 0) {
      uint32_t kbg = 0;
      for (int L = 0; L < nl; ++L) {
        const TcParams& p = layers[L];
        const ChainLayer ci = info[L];
        const int num_kb = p.ntaps * p.kchunks;
        const int bn = p.bn;
        const uint32_t tx_bytes = ((uint32_t)p.a_box_bytes + (uint32_t)(bn * BLOCK_K * 2)) * (uint32_t)NPL;
        if (lane == 0 && L + 1 < nl) {   // the next layer's descriptors: fetched long before their first use
          tma_prefetch_desc(&layers[L + 1].tmB);
          tma_prefetch_desc(&layers[L + 1].tmA[0]);
        }
        const bool nodeps = (ci.dep_a < 0 && ci.dep_r < 0);
        // the counters M tile m of this layer waits for: entry i of the list (input tiles first, then residual tiles);
        // returns the length of the list
        auto dep_of = [&](int m, int i, const int*& c, int& tgt) -> int {
          int r0, r1;
          chain_rows_of_tile(ci, m, r0, r1);
          int ia = 0, ib = -1, ja = 0, jb = -1, ta = 0, tr = 0;
          const int *ca = done, *cr = done;
          if (ci.dep_a >= 0) {   // input rows, in the producer's row numbering (its image height differs under a stride)
            const ChainLayer pa = info[ci.dep_a];
            int ra, rb;
            chain_input_rows(ci, pa, r0, r1, ra, rb);
            chain_tiles_of_rows(pa, ra, rb, ia, ib);
            ca = done + pa.done_off;
            ta = pa.target;
          }
          if (ci.dep_r >= 0) {   // the residual has this layer's geometry
            const ChainLayer pr = info[ci.dep_r];
            chain_tiles_of_rows(pr, r0, r1, ja, jb);
            cr = done + pr.done_off;
            tr = pr.target;
          }
          const int na = ib - ia + 1, nr = jb - ja + 1;
          if (i < na) {
            c = ca + ia + i;
            tgt = ta;
          } else {
            c = cr + ja + (i - na);
            tgt = tr;
          }
          return na + nr;
        };
        for (int u = chain_first_unit(cta, ci.ubase, G); u < ci.units; u += G) {
          const TileCoord tc_ = decode_unit<false>(p, u, 0, bn);
          bool ready = nodeps;
          for (int kb = 0; kb < num_kb; ++kb, ++kbg) {
            const uint32_t s = kbg % (uint32_t)stages;
            const uint32_t it = kbg / (uint32_t)stages;
            const int tap = kb / p.kchunks;
            const int kc = kb - tap * p.kchunks;
            uint8_t* sa = smem + (size_t)s * STAGE_BYTES;
            uint8_t* sb = sa + A_BYTES;
            if (lane == 0) {
              const long long t0 = stats ? clock64() : 0;
              mbar_wait(&empty_bar[s], (it & 1u) ^ 1u);
              if (stats) w1 += clock64() - t0;
              mbar_expect_tx(&full_bar[s], tx_bytes);
#pragma unroll
              for (int pl = 0; pl < NPL; ++pl)   // weights: constants, no dependency
                tma_load_3d(sb + pl * B_PLANE_BYTES, &p.tmB, &full_bar[s], kc * BLOCK_K + pl * p.cin, tc_.n0, tap);
            }
            if (!ready) {
              const long long tdep0 = stats ? clock64() : 0;
              __syncwarp();
              const int* c = done;
              int tgt = 0;
              const int n = dep_of(u / p.n_tiles, lane, c, tgt);
              for (int i = lane; i < n; i += 32) {
                if (i != lane) dep_of(u / p.n_tiles, i, c, tgt);
#ifdef YB_WATCHDOG
                const long long t0 = clock64();
#endif
                while (ld_acquire_gpu(c) < tgt) {
#ifdef YB_WATCHDOG
                  if (clock64() - t0 > 4000000000ll) asm volatile("trap;");
#endif
                }
              }
              __syncwarp();
              if (stats) w0 += clock64() - tdep0;
              fence_proxy_async_all();   // the tiles were written through the async proxy (TMA stores) and are read through it
              ready = true;
            }
            if (lane == 0) {
              const CUtensorMap* ma = &p.tmA[p.tap_map[tap]];
              const int ax = tc_.x0 + p.tap_dx[tap], ay = tc_.y0 + p.tap_dy[tap];
#pragma unroll
              for (int pl = 0; pl < NPL; ++pl)
                tma_load_4d(sa + pl * A_STAGE_BYTES, ma, &full_bar[s], kc * BLOCK_K + pl * p.cin, ax, ay, tc_.b);
            }
          }
        }
      }
      if (stats && lane == 0) {
        stats[cta * 8 + 0] = w0;
        stats[cta * 8 + 1] = w1;
      }
    }
  } else {
    // ===================== two MMA warpgroups: 64 rows of every tile each =====================
    const int cw = warp / 4 - 1;
    const int ct = threadIdx.x - 128;
    const int wq = warp & 3;
    const bool signaller = (threadIdx.x & 127) == 0;
    float acc[1][NPL][64];
    // thread 0 only: counter to bump once this thread's outstanding stores (the previous tile's) have completed
    int* pending = nullptr;
    auto flush_pending = [&]() {
      const long long t0 = stats ? clock64() : 0;
      bulk_wait_all();            // the stores have been performed, not just read out of shared memory
      if (stats) w0 += clock64() - t0;
      fence_proxy_async_all();
      red_release_gpu_add(pending, 1);
      pending = nullptr;
    };
    uint32_t kbg = 0, g = 0;
    for (int L = 0; L < nl; ++L) {
      const TcParams& p = layers[L];
      const int ubase = info[L].ubase, units = info[L].units, done_off = info[L].done_off;
      const int num_kb = p.ntaps * p.kchunks;
      const int n_tiles = p.n_tiles;
      const int bn = p.bn;
      for (int u = chain_first_unit(cta, ubase, G); u < units; u += G) {
        const TileCoord tc_ = decode_unit<false>(p, u, 0, bn);
        // The previous tile's completion signal waits for its stores; that is free when this tile's operands are not
        // ready yet (the warpgroups would idle anyway).  When they ARE ready the signal is deferred until after the
        // main loop -- safe, because ready operands mean this tile depends on nothing that could be waiting for it.
        if (ct == 0 && pending &&
            !mbar_test_wait(smem_u32(&full_bar[kbg % (uint32_t)stages]), (kbg / (uint32_t)stages) & 1u))
          flush_pending();
        if (bn == 128)
          mma_tile<128, 1, 2, SPLIT, false>(acc, smem, full_bar, empty_bar, stages, STAGE_BYTES, A_BYTES, B_PLANE_BYTES, kbg,
                                            num_kb, cw, signaller);
        else
          mma_tile<64, 1, 2, SPLIT, false>(acc, smem, full_bar, empty_bar, stages, STAGE_BYTES, A_BYTES, B_PLANE_BYTES, kbg,
                                           num_kb, cw, signaller);
        if (ct == 0 && pending) flush_pending();
        EpiArgs e;
        e.tmY = &p.tmY;
        e.tmR = &p.tmR;
        e.res_full_bar = nullptr;
        e.out_base = out_base;
        e.res_base = nullptr;
        e.bias = p.bias;
        e.res_g = p.residual ? p.residual + (size_t)tc_.x0 * (size_t)(NPL * p.Cout) + tc_.n0 : nullptr;   // flattened layouts only
        e.res_pix_stride = NPL * p.Cout;
        e.res_tx = 0;   // (no staged residual in a chain)
        e.Wo = p.Wo;
        e.Cout = p.Cout;
        e.n0 = tc_.n0;
        e.x0 = tc_.x0;
        e.y0 = tc_.y0;
        e.b = tc_.b;
        e.nchunks = bn / 64;
        e.nbuf = SPLIT ? 1 : 2;
        e.out_scale = p.out_scale;
        if (bn == 128) epi_staged_act<SPLIT, 128, 1, 2>(p.act, p.res_after_act, acc, e, false, g, cw, ct, lane, wq);
        else epi_staged_act<SPLIT, 64, 1, 2>(p.act, p.res_after_act, acc, e, false, g, cw, ct, lane, wq);
        if (ct == 0) pending = done + done_off + u / n_tiles;
      }
    }
    if (ct == 0) {
      if (pending) flush_pending();
      bulk_wait_read<0>();
      if (stats) {
        stats[cta * 8 + 4] = w0;
        stats[cta * 8 + 6] = clock64() - t_kernel0;
      }
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
int floordiv(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }

}  // namespace

// SMs of the current device (132 on an H100 SXM): the persistent grids hold one CTA (or pair) per SM, and the stream-K
// workspace one slot per CTA
int device_sms() {
  static std::atomic<int> cached[64] = {};
  int dev = 0;
  YB_CHECK_CUDA(cudaGetDevice(&dev));
  int n = cached[dev & 63].load();
  if (n <= 0) {
    YB_CHECK_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
    cached[dev & 63].store(n);
  }
  return n;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                    CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                    CUtensorMapFloatOOBfill);

namespace {
PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  YB_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres));
  YB_REQUIRE(qres == cudaDriverEntryPointSuccess && ptr, "cuTensorMapEncodeTiled not available from the driver");
  fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  return fn;
}

}  // namespace

void tc::encode_map_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                const uint32_t* box, int swizzle_bytes) {
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    YB_REQUIRE(box[i] >= 1 && box[i] <= 256, "tensor map: box dim out of range");
  }
  for (int i = 0; i + 1 < rank; ++i) {
    gstr[i] = strides_bytes[i];
    YB_REQUIRE(strides_bytes[i] % 16 == 0, "tensor map: stride must be a multiple of 16 bytes");
  }
  YB_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "tensor map: base must be 16-byte aligned");
  CUresult r = get_encode_fn()(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base),
                               gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                               swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    throw Error(YB_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
}


struct TcConvPlan {
  TcParams prm;
  int split = 0;
  int sk = 0;           // stream-K requested (effective once a workspace is attached: prm.sk)
  int BN = 128;
  int pair = 0;
  int epi_groups = 1;   // H: MMA warpgroups per CTA (each owns 2/H of the tile's 64-row halves)
  int pdl_friendly = 0; // sized so that two CTAs (this kernel's and the next layer's) fit on one SM
  int chain = 0;        // planned for the chain kernel
  int flat = 0;         // 1x1 / stride 1 / dense: all pixels of the batch on one axis
  int B = 0, Ho = 0, Wo = 0;   // the problem's output geometry (prm.Ho / prm.Wo are the flattened view's)
  int Hi = 0, Wi = 0, stride = 1, pad = 0, KH = 1;
  dim3 grid;
  size_t smem_bytes = 0;
};

bool tc_conv_supported(const ConvProblem& p) {
  if (p.x_nchw_f32) return false;
  if (p.Cin % BLOCK_K != 0) return false;
  if (p.KH * p.KW > MAX_TAPS) return false;
  if (p.stride != 1 && p.stride != 2) return false;
  if (p.Cout < 1) return false;
  return true;
}

// spatial tile tw x th <= 128 accumulator rows with the best fill (ties: the wider tile)
static void choose_tile(int Wov, int Hov, int& best_tw, int& best_th) {
  best_tw = 1;
  best_th = 1;
  double best_eff = -1.0;
  for (int tw = 1; tw <= std::min(Wov, 128); ++tw) {
    int th = std::min(Hov, 128 / tw);
    if (th < 1) continue;
    if (tw > 256 || th > 256) continue;
    long long tiles = (long long)ceil_div(Wov, tw) * ceil_div(Hov, th);
    double eff = (double)Wov * Hov / ((double)tiles * 128.0);
    if (eff > best_eff + 1e-9 || (eff > best_eff - 1e-9 && tw > best_tw)) {
      best_eff = eff;
      best_tw = tw;
      best_th = th;
    }
  }
}

// Host mirror of the chain kernel's dependency arithmetic for ONE consumer layer (a k x k conv, stride, pad, on a
// B x Hin x Win input written by a producer layer that is flattened (1x1 stride 1) or not): the tilings both layers
// would get and, for consumer M tile m, the inclusive range of producer M tiles the kernel would wait for.
// out[0..5] = consumer flat, tw, th, tiles_x, tiles_y, m_tiles; out[6..11] = producer flat, tw, th, tiles_x, tiles_y,
// m_tiles; out[12], out[13] = first, last producer tile.  No device needed.
void tc_chain_debug_deps(int B, int Hin, int Win, int k, int stride, int pad, int producer_flat, int m, int32_t* out) {
  YB_REQUIRE(B >= 1 && Hin >= 1 && Win >= 1 && (k == 1 || k == 3) && (stride == 1 || stride == 2) && pad >= 0 && out,
             "chain_debug_deps: bad argument");
  const int Ho = conv_out(Hin, k, stride, pad), Wo = conv_out(Win, k, stride, pad);
  YB_REQUIRE(Ho >= 1 && Wo >= 1, "chain_debug_deps: empty output");
  auto layer = [&](int flat, int H, int W, int s, int p, int kh) {
    ChainLayer c = {};
    c.flat = flat;
    c.W = W;
    c.H = H;
    c.rows = B * H;
    const int Wov = flat ? B * H * W : W, Hov = flat ? 1 : H;
    choose_tile(Wov, Hov, c.tw, c.th);
    c.tiles_x = ceil_div(Wov, c.tw);
    c.tiles_y = ceil_div(Hov, c.th);
    c.stride = s;
    c.pad = p;
    c.kh = kh;
    return c;
  };
  const ChainLayer ci = layer((k == 1 && stride == 1 && pad == 0) ? 1 : 0, Ho, Wo, stride, pad, k);
  const ChainLayer pa = layer(producer_flat ? 1 : 0, Hin, Win, 1, 0, 1);
  const int cm = ci.tiles_x * ci.tiles_y * (ci.flat ? 1 : B), pm = pa.tiles_x * pa.tiles_y * (pa.flat ? 1 : B);
  YB_REQUIRE(m >= 0 && m < cm, "chain_debug_deps: tile out of range");
  int r0, r1, ra, rb, ia, ib;
  chain_rows_of_tile(ci, m, r0, r1);
  chain_input_rows(ci, pa, r0, r1, ra, rb);
  chain_tiles_of_rows(pa, ra, rb, ia, ib);
  const int32_t v[14] = {ci.flat, ci.tw, ci.th, ci.tiles_x, ci.tiles_y, cm, pa.flat, pa.tw, pa.th, pa.tiles_x, pa.tiles_y, pm, ia, ib};
  for (int i = 0; i < 14; ++i) out[i] = v[i];
}

TcConvPlan* tc_conv_plan_create(const ConvProblem& p, const __half* w_packed, const TcTiling& want) {
  YB_REQUIRE(tc_conv_supported(p), "tc_conv: unsupported problem");
  YB_REQUIRE(p.Ho >= 1 && p.Ho == conv_out(p.H, p.KH, p.stride, p.pad), "tc_conv: bad Ho");
  YB_REQUIRE(p.Wo >= 1 && p.Wo == conv_out(p.W, p.KW, p.stride, p.pad), "tc_conv: bad Wo");
  auto* plan = new TcConvPlan();
  TcParams& q = plan->prm;
  memset(&q, 0, sizeof(q));
  const int s = p.stride;
  q.ntaps = p.KH * p.KW;
  q.kchunks = p.Cin / BLOCK_K;
  const int split = p.split ? 1 : 0;
  const int npl = split ? 2 : 1;       // fp16 planes per operand / activation
  plan->split = split;
  q.split = split;
  q.cin = p.Cin;
  q.out_scale = split ? p.out_scale : 1.f;

  // ---- geometry: can the whole problem be flattened into one pixel axis? (1x1, stride 1, dense out)
  const bool dense_out = (p.y_batch_stride == (int64_t)p.Ho * p.Wo * p.y_pix_stride);
  YB_REQUIRE(!split || p.y_f32 || p.nseg > 0 || p.y_pix_stride >= 2 * p.Cout, "tc_conv: split outputs need 2*Cout halfs per pixel");
  const bool flat = (q.ntaps == 1 && s == 1 && p.pad == 0 && dense_out);
  int Bv = p.B, Hov = p.Ho, Wov = p.Wo;
  if (flat) {
    Wov = p.B * p.Ho * p.Wo;
    Hov = 1;
    Bv = 1;
  }
  // ---- spatial tile (tw x th <= 128) with the best fill
  int best_tw = 1, best_th = 1;
  choose_tile(Wov, Hov, best_tw, best_th);
  plan->flat = flat ? 1 : 0;
  plan->B = p.B;
  plan->Ho = p.Ho;
  plan->Wo = p.Wo;
  plan->Hi = p.H;
  plan->Wi = p.W;
  plan->stride = p.stride;
  plan->pad = p.pad;
  plan->KH = p.KH;
  q.tw = best_tw;
  q.th = best_th;
  q.tiles_x = ceil_div(Wov, q.tw);
  q.tiles_y = ceil_div(Hov, q.th);
  q.Ho = Hov;
  q.Wo = Wov;
  q.Cout = p.Cout;
  q.a_box_bytes = q.tw * q.th * BLOCK_K * 2;
  const long long m_tiles = (long long)q.tiles_x * q.tiles_y * Bv;

  // ---- epilogue mode: fp16 NHWC outputs with 16-byte aligned rows go through smem + TMA store
  const int esz = p.y_f32 ? 4 : 2;
  const int vec_elems = 16 / esz;
  bool vec_ok = (p.y_pix_stride % vec_elems == 0) && (p.y_batch_stride % vec_elems == 0) &&
                ((reinterpret_cast<uintptr_t>(p.y) & 15) == 0);
  if (p.residual) vec_ok = vec_ok && (p.Cout % 8 == 0) && ((reinterpret_cast<uintptr_t>(p.residual) & 15) == 0);
  q.vec_ok = vec_ok ? 1 : 0;
  q.epi_tma = (!p.y_f32 && vec_ok && p.Cout % 8 == 0 && p.nseg == 0) ? 1 : 0;
  // split: a 64-channel hi box must not run into the lo plane of the same pixel (nothing clips it there)
  if (split && q.epi_tma && p.Cout % 64 != 0) q.epi_tma = 0;
  // the staged epilogue has an act-then-add instance for LeakyReLU (Darknet blocks) only (epi_staged_act)
  YB_REQUIRE(!q.epi_tma || !p.res_after_act || p.act == ACT_LEAKY || p.act == ACT_NONE,
             "tc_conv: a residual after the activation needs LeakyReLU (or none) with a half-precision output");
  // the staged epilogue moves 64-channel boxes: a CTA must own at least 64 output channels
  const int bn_min = q.epi_tma ? 64 : 32;

  // ---- N tile: minimise waves * (BN + fixed cost)
  const int sms = device_sms();
  {
    const int cands[4] = {256, 128, 64, 32};
    double best = 1e30;
    int bn_best = 32;
    for (int i = 0; i < 4; ++i) {
      int bn = cands[i];
      if (bn < bn_min) continue;
      if (bn > bn_min && bn >= 2 * p.Cout) continue;  // more than half the tile would be padding
      long long ctas = m_tiles * ceil_div(p.Cout, bn);
      long long waves = (ctas + sms - 1) / sms;
      double cost = (double)waves * (bn + 64);
      if (cost < best - 1e-9) {
        best = cost;
        bn_best = bn;
      }
    }
    plan->BN = bn_best;
    if (want.bn == 32 || want.bn == 64 || want.bn == 128 || want.bn == 256)
      plan->BN = std::max(want.bn, bn_min);
  }
  // ---- CTA pairs: two adjacent M tiles per (cluster of 2), each CTA loads half of the weight tile for both
  const int pair = (want.pair > 0 && m_tiles >= 2 && plan->BN >= 64) ? 1 : 0;
  // PDL-friendly plan: <= ~108 KB of shared memory and one MMA warpgroup, so that a CTA of the NEXT layer can become
  // resident beside it and overlap its prologue + first weight tiles
  const int pdlf = (want.pdl_friendly > 0 && !pair && !split) ? 1 : 0;
  // ---- MMA warpgroups: the accumulators of a thread (npl * BN / H fp32 registers) must stay <= 128
  int H = (want.mma_groups == 2 && plan->BN >= 64 && !pdlf) ? 2 : 1;
  if (npl * plan->BN > 128 && !pdlf) H = 2;
  while (npl * plan->BN / H > 128 && plan->BN > std::max(bn_min, pair ? 64 : 32)) plan->BN /= 2;
  YB_REQUIRE(npl * plan->BN / H <= 128, "tc_conv: accumulator tile exceeds the register budget");
  plan->epi_groups = H;
  plan->pdl_friendly = pdlf;
  const int BN = plan->BN;
  q.bn = BN;
  plan->pair = pair;
  q.pair = pair;
  q.nb = Bv;
  const int stage_bytes = npl * (A_STAGE_BYTES + BN * BLOCK_K * 2);   // a pair CTA receives the whole weight tile too
  // ---- persistent grid + shared-memory layout: [pipeline stages][2 x 16 KB out tiles][2 x 16 KB residual tiles]
  q.m_tiles = (int)m_tiles;
  q.n_tiles = ceil_div(p.Cout, BN);
  const int num_tiles = (pair ? (q.m_tiles + 1) / 2 : q.m_tiles) * q.n_tiles;   // work units (pairs of M tiles when paired)
  const int max_grid = pair ? sms / 2 : sms;
  int grid = std::min(num_tiles, want.grid > 0 ? (pair ? std::max(1, want.grid / 2) : want.grid) : max_grid);
  if (pair) grid = std::min(grid, max_grid);
  // stream-K: one share of the k-block iterations per SM (cluster), whatever the unit count -- worth it only when the
  // units do not fill whole waves; needs the staged (TMA) epilogue and co-resident CTAs (<= one per SM)
  const long long total_it = (long long)num_tiles * q.ntaps * q.kchunks;
  int sk = (want.stream_k > 0 && q.epi_tma && !(want.pdl_friendly > 0)) ? 1 : 0;
  if (sk) {
    const int gsk = std::min<long long>(want.grid > 0 ? grid : max_grid, total_it);
    if (gsk <= 1 || num_tiles % gsk == 0) sk = 0;   // whole waves already: nothing to balance
    else grid = gsk;
  }
  plan->sk = sk;
  const int tiles_per_cta = sk ? 2 : ceil_div(num_tiles, grid);
  // staging: 2 x 16 KB (two fp16 buffers, or one buffer of a hi and a lo tile); the direct (fp32) epilogue stores
  // straight from the accumulator registers
  const int out_bytes = q.epi_tma ? 2 * A_STAGE_BYTES : 0;
  plan->chain = want.chain > 0 ? 1 : 0;
  q.res_direct = ((split || plan->chain) && H == 2 && p.residual && flat && q.epi_tma) ? 1 : 0;
  const int res_bytes = (q.epi_tma && p.residual && !q.res_direct) ? 2 * A_STAGE_BYTES : 0;
  int stages = std::min(MAX_STAGES, ((pdlf ? 108 : 225) * 1024 - out_bytes - res_bytes) / stage_bytes);
  if (stages < 1 && pdlf) {   // does not fit in half an SM: an ordinary plan
    plan->pdl_friendly = 0;
    stages = std::min(MAX_STAGES, (225 * 1024 - out_bytes - res_bytes) / stage_bytes);
  }
  YB_REQUIRE(stages >= 1, "tc_conv: tile does not fit in shared memory");
  if (want.stages > 0) stages = std::min(stages, want.stages);
  stages = std::max(1, std::min(stages, q.ntaps * q.kchunks * tiles_per_cta));
  q.stages = stages;
  q.out_off = stages * stage_bytes;
  q.res_off = q.out_off + out_bytes;
  plan->smem_bytes = (size_t)q.res_off + res_bytes + 1024;
  if (plan->pdl_friendly && plan->smem_bytes > (size_t)112 * 1024) plan->pdl_friendly = 0;   // does not fit twice: plain plan
  q.pdl = plan->pdl_friendly;
  plan->grid = dim3((unsigned)(pair ? 2 * grid : grid), 1, 1);

  // ---- A tensor maps
  const __half* x = reinterpret_cast<const __half*>(p.x);
  const uint64_t CinP = (uint64_t)npl * p.Cin;    // halfs per input pixel (both planes)
  const uint64_t CoutP = (uint64_t)npl * p.Cout;  // halfs per residual pixel
  if (flat) {
    uint64_t dims[4] = {CinP, (uint64_t)Wov, 1, 1};
    uint64_t str[3] = {CinP * 2, (uint64_t)Wov * CinP * 2, (uint64_t)Wov * CinP * 2};
    uint32_t box[4] = {(uint32_t)BLOCK_K, (uint32_t)q.tw, (uint32_t)q.th, 1};
    encode_map_f16(&q.tmA[0], x, 4, dims, str, box);
    q.tap_map[0] = 0;
    q.tap_dx[0] = 0;
    q.tap_dy[0] = 0;
  } else {
    bool used[4] = {false, false, false, false};
    for (int r = 0; r < p.KH; ++r)
      for (int c = 0; c < p.KW; ++c) {
        int qy = r - p.pad, qx = c - p.pad;
        int py = ((qy % s) + s) % s, px = ((qx % s) + s) % s;
        int tap = r * p.KW + c;
        q.tap_map[tap] = py * s + px;
        q.tap_dy[tap] = floordiv(qy - py, s);
        q.tap_dx[tap] = floordiv(qx - px, s);
        used[py * s + px] = true;
      }
    // a stride-2 phase is empty on a one-pixel side (H == 1: no odd rows): its taps read only the conv's zero padding.
    // They load from phase 0 (never empty) at a row offset past its last row instead: TMA zero-fills a box that lies
    // wholly out of bounds and still counts its full bytes, so they add exactly zero with no kernel branch.
    const int H0 = (p.H + s - 1) / s;
    for (int tap = 0; tap < q.ntaps; ++tap) {
      const int ph = q.tap_map[tap], py = ph / s, px = ph % s;
      if (p.H - py >= 1 && p.W - px >= 1) continue;
      q.tap_map[tap] = 0;
      q.tap_dy[tap] = H0;
      q.tap_dx[tap] = 0;
      used[0] = true;
    }
    for (int py = 0; py < s; ++py)
      for (int px = 0; px < s; ++px) {
        if (!used[py * s + px]) continue;
        int Hv = (p.H - py + s - 1) / s, Wv = (p.W - px + s - 1) / s;
        if (Hv < 1 || Wv < 1) continue;   // no tap reads it (remapped above)
        const __half* base = x + ((size_t)py * p.W + px) * CinP;
        uint64_t dims[4] = {CinP, (uint64_t)Wv, (uint64_t)Hv, (uint64_t)p.B};
        uint64_t str[3] = {(uint64_t)s * CinP * 2, (uint64_t)s * p.W * CinP * 2,
                           (uint64_t)p.H * p.W * CinP * 2};
        uint32_t box[4] = {(uint32_t)BLOCK_K, (uint32_t)q.tw, (uint32_t)q.th, 1};
        encode_map_f16(&q.tmA[py * s + px], base, 4, dims, str, box);
      }
  }
  // ---- B tensor map: [tap][Cout][Cin]
  {
    uint64_t dims[3] = {CinP, (uint64_t)p.Cout, (uint64_t)q.ntaps};
    uint64_t str[2] = {CinP * 2, (uint64_t)p.Cout * CinP * 2};
    uint32_t box[3] = {(uint32_t)BLOCK_K, (uint32_t)(pair ? BN / 2 : BN), 1};   // a pair CTA loads half a weight tile
    encode_map_f16(&q.tmB, w_packed, 3, dims, str, box);
  }
  // ---- epilogue
  q.y = p.y;
  q.bias = p.bias;
  q.residual = reinterpret_cast<const __half*>(p.residual);
  q.y_f32 = p.y_f32;
  q.act = p.act;
  q.res_after_act = p.res_after_act;
  q.nseg = p.nseg;
  for (int i = 0; i < p.nseg && i < 3; ++i) {
    q.seg_begin[i] = p.seg_begin[i];
    q.seg_end[i] = p.seg_end[i];
    q.seg_ps[i] = p.seg_ps[i];
    q.seg_act[i] = p.seg_act[i];
    q.seg_bs[i] = p.seg_bs[i];
    q.seg_y[i] = p.seg_y[i];
  }
  q.y_pix_stride = p.y_pix_stride;
  if (flat) {
    q.y_batch_stride = 0;
    q.res_batch_stride = 0;
  } else {
    q.y_batch_stride = p.y_batch_stride;
    q.res_batch_stride = (long long)p.Ho * p.Wo * p.Cout;   // pixels * Cout; the kernel scales by the plane count
  }
  if (q.epi_tma) {
    // output / residual tile maps: same geometry as the accumulator tile, 64-channel boxes
    uint32_t box[4] = {(uint32_t)BLOCK_K, (uint32_t)q.tw, (uint32_t)q.th, 1};
    if (flat) {
      uint64_t dims[4] = {CoutP, (uint64_t)Wov, 1, 1};
      uint64_t ystr[3] = {(uint64_t)p.y_pix_stride * 2, (uint64_t)Wov * p.y_pix_stride * 2, (uint64_t)Wov * p.y_pix_stride * 2};
      encode_map_f16(&q.tmY, p.y, 4, dims, ystr, box);
      if (p.residual) {
        uint64_t rstr[3] = {CoutP * 2, (uint64_t)Wov * CoutP * 2, (uint64_t)Wov * CoutP * 2};
        encode_map_f16(&q.tmR, p.residual, 4, dims, rstr, box);
      }
    } else {
      uint64_t dims[4] = {CoutP, (uint64_t)p.Wo, (uint64_t)p.Ho, (uint64_t)p.B};
      uint64_t ystr[3] = {(uint64_t)p.y_pix_stride * 2, (uint64_t)p.Wo * p.y_pix_stride * 2, (uint64_t)p.y_batch_stride * 2};
      encode_map_f16(&q.tmY, p.y, 4, dims, ystr, box);
      if (p.residual) {
        uint64_t rstr[3] = {CoutP * 2, (uint64_t)p.Wo * CoutP * 2, (uint64_t)p.Ho * p.Wo * CoutP * 2};
        encode_map_f16(&q.tmR, p.residual, 4, dims, rstr, box);
      }
    }
  }
  return plan;
}

void tc_conv_plan_destroy(TcConvPlan* plan) { delete plan; }
void tc_conv_plan_set_pdl(TcConvPlan* plan, int enable) { plan->prm.pdl = (enable && !plan->pair) ? 1 : 0; }
TcTiling tc_conv_plan_tiling(const TcConvPlan* plan) {
  TcTiling t;
  t.bn = plan->BN;
  t.stages = plan->prm.stages;
  t.grid = (int)plan->grid.x;
  t.pair = plan->pair;
  t.mma_groups = plan->epi_groups;
  t.pdl_friendly = plan->pdl_friendly;
  t.stream_k = plan->sk;
  t.chain = plan->chain;
  return t;
}
std::string tc_tiling_str(const TcTiling& t) {
  return "BN=" + std::to_string(t.bn) + " st=" + std::to_string(t.stages) + " g=" + std::to_string(t.grid) +
         (t.pair ? " pair" : "") + (t.mma_groups == 2 ? " epi2" : "") + (t.pdl_friendly ? " pdlf" : "") +
         (t.stream_k ? " sk" : "") + (t.chain ? " chain" : "");
}
// one slot per SM of the current device (a stream-K grid has at most one CTA per SM)
size_t tc_conv_sk_workspace_bytes() { return (size_t)device_sms() * BLOCK_M * 256 * sizeof(float) + device_sms() * 2 * sizeof(int); }
// ws: tc_conv_sk_workspace_bytes() of device memory whose LAST device_sms() * 2 ints (the flags) are zero; kernels that share a
// workspace must be stream-ordered (each launch leaves the flags zero again)
void tc_conv_plan_set_sk_workspace(TcConvPlan* plan, void* ws) {
  plan->prm.sk = (plan->sk && ws) ? 1 : 0;
  plan->prm.sk_ws = reinterpret_cast<float*>(ws);
  plan->prm.sk_flags = reinterpret_cast<int*>(reinterpret_cast<char*>(ws) + (size_t)device_sms() * BLOCK_M * 256 * sizeof(float));
}

template <int BN, bool PAIR, int H, bool SPLIT>
static void launch_bn(const TcConvPlan* plan, cudaStream_t stream) {
  static PerDeviceOnce attr;
  if (attr.first())
    YB_CHECK_CUDA(cudaFuncSetAttribute(tc_conv_kernel<BN, PAIR, H, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)(226 * 1024)));
  constexpr int THREADS = 128 * (1 + H);
  if (plan->prm.pdl || PAIR) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = plan->grid;
    cfg.blockDim = dim3(THREADS);
    cfg.dynamicSmemBytes = plan->smem_bytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    int na = 0;
    if (PAIR) {
      attr[na].id = cudaLaunchAttributeClusterDimension;
      attr[na].val.clusterDim.x = 2;
      attr[na].val.clusterDim.y = 1;
      attr[na].val.clusterDim.z = 1;
      ++na;
    } else {
      attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      attr[na].val.programmaticStreamSerializationAllowed = 1;
      ++na;
    }
    cfg.attrs = attr;
    cfg.numAttrs = na;
    YB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, tc_conv_kernel<BN, PAIR, H, SPLIT>, plan->prm));
  } else {
    tc_conv_kernel<BN, PAIR, H, SPLIT><<<plan->grid, THREADS, plan->smem_bytes, stream>>>(plan->prm);
  }
}

// the (BN, warpgroups) combinations whose accumulators fit in 128 registers per thread (the plan never picks others)
template <int BN, bool PAIR, bool SPLIT>
static void launch_h(const TcConvPlan* plan, cudaStream_t stream) {
  constexpr int NPL = SPLIT ? 2 : 1;
  if (plan->epi_groups == 2) {
    if constexpr (NPL * BN / 2 <= 128) launch_bn<BN, PAIR, 2, SPLIT>(plan, stream);
    else YB_REQUIRE(false, "tc_conv: N tile too wide for two MMA warpgroups");
  } else {
    if constexpr (NPL * BN <= 128) launch_bn<BN, PAIR, 1, SPLIT>(plan, stream);
    else YB_REQUIRE(false, "tc_conv: N tile too wide for one MMA warpgroup");
  }
}

template <bool SPLIT>
static void launch_s(const TcConvPlan* plan, cudaStream_t stream) {
  if (plan->pair) {
    switch (plan->BN) {
      case 256: launch_h<256, true, SPLIT>(plan, stream); break;
      case 128: launch_h<128, true, SPLIT>(plan, stream); break;
      case 64: launch_h<64, true, SPLIT>(plan, stream); break;
      default: YB_REQUIRE(false, "tc_conv: bad BN for a CTA pair");
    }
  } else {
    switch (plan->BN) {
      case 256: launch_h<256, false, SPLIT>(plan, stream); break;
      case 128: launch_h<128, false, SPLIT>(plan, stream); break;
      case 64: launch_h<64, false, SPLIT>(plan, stream); break;
      case 32: launch_h<32, false, SPLIT>(plan, stream); break;
      default: YB_REQUIRE(false, "tc_conv: bad BN");
    }
  }
}

// ---------------------------------------------------------------------------------------------
// chains
// ---------------------------------------------------------------------------------------------
struct TcChain {
  int nl = 0, split = 0, grid = 0, n_done = 0;
  size_t smem_bytes = 0;
  TcParams* d_layers = nullptr;
  ChainLayer* d_info = nullptr;
  int* d_done = nullptr;
  long long* d_stats = nullptr;   // diagnostics (YB_CHAIN_STATS=1)
};

// a plan the chain kernel can run: its tile shape (BN = 128 or 64, two MMA warpgroups, staged epilogue) and nothing the
// chain does not implement (pairs, stream-K, staged residual, partial N tiles)
bool tc_conv_plan_chainable(const TcConvPlan* pl) {
  const TcParams& q = pl->prm;
  return (pl->BN == 128 || pl->BN == 64) && !pl->pair && pl->epi_groups == 2 && !pl->sk && !pl->pdl_friendly && q.epi_tma &&
         q.nseg == 0 && q.Cout % pl->BN == 0 && (!q.residual || q.res_direct) && (q.act == ACT_RELU || q.act == ACT_NONE || q.act == ACT_LEAKY);
}

// dep_a[i] / dep_r[i]: index (< i) of the plan that writes plan i's input / residual, -1 for a tensor that is complete
// before the launch (or, for the residual, one whose completion the input dependency already implies)
TcChain* tc_chain_create(const std::vector<const TcConvPlan*>& plans, const std::vector<int>& dep_a, const std::vector<int>& dep_r) {
  YB_REQUIRE(!plans.empty() && plans.size() == dep_a.size() && plans.size() == dep_r.size(), "tc_chain: empty chain");
  const TcConvPlan* p0 = plans[0];
  std::vector<TcParams> lp;
  std::vector<ChainLayer> li;
  int ubase = 0, done_off = 0;
  for (size_t i = 0; i < plans.size(); ++i) {
    const TcConvPlan* pl = plans[i];
    YB_REQUIRE(tc_conv_plan_chainable(pl), "tc_chain: plan not chainable");
    YB_REQUIRE(pl->split == p0->split, "tc_chain: the layers of a chain share one precision mode");
    YB_REQUIRE(pl->B == p0->B, "tc_chain: the layers of a chain share one batch size");
    YB_REQUIRE(dep_a[i] < (int)i && dep_r[i] < (int)i, "tc_chain: dependencies point backwards");
    YB_REQUIRE(dep_r[i] < 0 || (plans[dep_r[i]]->Ho == pl->Ho && plans[dep_r[i]]->Wo == pl->Wo), "tc_chain: residual geometry");
    YB_REQUIRE(dep_a[i] < 0 || (plans[dep_a[i]]->Ho == pl->Hi && plans[dep_a[i]]->Wo == pl->Wi), "tc_chain: input geometry");
    ChainLayer c = {};
    c.ubase = ubase;
    c.units = pl->prm.m_tiles * pl->prm.n_tiles;
    c.flat = pl->flat;
    c.W = pl->Wo;
    c.H = pl->Ho;
    c.rows = pl->B * pl->Ho;
    c.tw = pl->prm.tw;
    c.th = pl->prm.th;
    c.tiles_x = pl->prm.tiles_x;
    c.tiles_y = pl->prm.tiles_y;
    c.done_off = done_off;
    c.target = pl->prm.n_tiles;   // each (M tile, N tile) adds 1 once its stores have completed
    c.dep_a = dep_a[i];
    c.dep_r = dep_r[i];
    c.stride = pl->stride;
    c.pad = pl->pad;
    c.kh = pl->KH;
    ubase += c.units;
    done_off += pl->prm.m_tiles;
    lp.push_back(pl->prm);
    li.push_back(c);
  }
  auto* ch = new TcChain();
  ch->nl = (int)plans.size();
  ch->split = p0->split;
  ch->n_done = done_off;
  {
    const int npl = p0->split ? 2 : 1;
    ch->smem_bytes = (size_t)chain_stages(p0->split != 0) * npl * (A_STAGE_BYTES + 128 * BLOCK_K * 2) +
                     (size_t)(p0->split ? 1 : 2) * npl * A_STAGE_BYTES + 1024;
  }
  const int sms = device_sms();
  ch->grid = std::min(sms, ubase);   // one CTA per SM (the shared memory of a CTA sees to that): all co-resident
  try {
    YB_CHECK_CUDA(cudaMalloc(&ch->d_layers, lp.size() * sizeof(TcParams)));
    YB_CHECK_CUDA(cudaMalloc(&ch->d_info, li.size() * sizeof(ChainLayer)));
    YB_CHECK_CUDA(cudaMalloc(&ch->d_done, (size_t)done_off * sizeof(int)));
    YB_CHECK_CUDA(cudaMemcpy(ch->d_layers, lp.data(), lp.size() * sizeof(TcParams), cudaMemcpyHostToDevice));
    YB_CHECK_CUDA(cudaMemcpy(ch->d_info, li.data(), li.size() * sizeof(ChainLayer), cudaMemcpyHostToDevice));
  } catch (...) {
    tc_chain_destroy(ch);
    throw;
  }
  return ch;
}
void tc_chain_destroy(TcChain* ch) {
  if (!ch) return;
  cudaFree(ch->d_layers);
  cudaFree(ch->d_info);
  cudaFree(ch->d_done);
  cudaFree(ch->d_stats);
  delete ch;
}
int tc_chain_layers(const TcChain* ch) { return ch->nl; }

template <bool SPLIT>
static void launch_chain_t(const TcChain* ch, cudaStream_t stream) {
  static PerDeviceOnce attr;
  if (attr.first())
    YB_CHECK_CUDA(cudaFuncSetAttribute(tc_chain_kernel<SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)ch->smem_bytes));   // (one size per precision mode)
  // Cooperative launch: the grid starts only when ALL its CTAs can be resident at once.  The tile dependencies make CTAs
  // wait for each other, so a partially scheduled grid (two chains from different streams sharing the SMs) could deadlock.
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)ch->grid);
  cfg.blockDim = dim3(384);
  cfg.dynamicSmemBytes = ch->smem_bytes;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative;
  at[0].val.cooperative = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  YB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, tc_chain_kernel<SPLIT>, (const TcParams*)ch->d_layers, (const ChainLayer*)ch->d_info,
                                   ch->nl, ch->d_done, ch->d_stats));
}

// diagnostics: one launch with the wait counters on, averaged over the CTAs -> stderr
void tc_chain_print_stats(TcChain* ch, const char* name) {
  const int G = ch->grid;
  YB_CHECK_CUDA(cudaMalloc(&ch->d_stats, (size_t)G * 8 * sizeof(long long)));
  YB_CHECK_CUDA(cudaMemset(ch->d_stats, 0, (size_t)G * 8 * sizeof(long long)));
  launch_tc_chain(ch, 0, nullptr);
  YB_CHECK_CUDA(cudaDeviceSynchronize());
  std::vector<long long> hs((size_t)G * 8);
  YB_CHECK_CUDA(cudaMemcpy(hs.data(), ch->d_stats, hs.size() * sizeof(long long), cudaMemcpyDeviceToHost));
  cudaFree(ch->d_stats);
  ch->d_stats = nullptr;
  double avg[8] = {}, mx[8] = {};
  for (int c = 0; c < G; ++c)
    for (int k = 0; k < 8; ++k) {
      avg[k] += (double)hs[(size_t)c * 8 + k] / G;
      mx[k] = std::max(mx[k], (double)hs[(size_t)c * 8 + k]);
    }
  const double tot = avg[6] > 0 ? avg[6] : 1.0;
  fprintf(stderr,
          "[yolact_b200] chain stats %s: kernel %.0f kcyc/CTA; share of it spent waiting (avg over CTAs / max): producer deps %.1f%% / %.1f%%, "
          "producer ring slot %.1f%%, store completion before a signal %.1f%% / %.1f%%\n",
          name, tot / 1e3, 100 * avg[0] / tot, 100 * mx[0] / tot, 100 * avg[1] / tot, 100 * avg[4] / tot, 100 * mx[4] / tot);
}

// Can a chain launch be captured into a CUDA graph and replayed on this driver?  (One trial per process.)
bool tc_chain_graph_ok(const TcChain* ch) {
  static std::atomic<int> cached{-1};   // (executors of different handles may be built from different threads)
  if (cached.load() >= 0) return cached.load() != 0;
  bool ok = false;
  cudaStream_t s = nullptr;
  cudaGraph_t g = nullptr;
  cudaGraphExec_t ge = nullptr;
  if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) == cudaSuccess) {
    if (cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
      try {
        launch_tc_chain(ch, s, nullptr);
      } catch (const Error&) {
      }
      if (cudaStreamEndCapture(s, &g) == cudaSuccess && g && cudaGraphInstantiate(&ge, g, 0) == cudaSuccess)
        ok = (cudaGraphLaunch(ge, s) == cudaSuccess) && (cudaStreamSynchronize(s) == cudaSuccess);
    }
  }
  if (ge) cudaGraphExecDestroy(ge);
  if (g) cudaGraphDestroy(g);
  if (s) cudaStreamDestroy(s);
  cudaGetLastError();
  cached.store(ok ? 1 : 0);
  return ok;
}
void launch_tc_chain(const TcChain* ch, cudaStream_t stream, LaunchCounter* lc) {
  YB_CHECK_CUDA(cudaMemsetAsync(ch->d_done, 0, (size_t)ch->n_done * sizeof(int), stream));   // (a memset node in the captured graph)
  if (ch->split) launch_chain_t<true>(ch, stream); else launch_chain_t<false>(ch, stream);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

void launch_tc_conv(const TcConvPlan* plan, cudaStream_t stream, LaunchCounter* lc) {
  if (plan->split) launch_s<true>(plan, stream); else launch_s<false>(plan, stream);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

}  // namespace yb
