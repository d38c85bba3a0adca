// Sparse-conv gather-GEMM on wgmma, fp16 hi/lo split rows ("H16"), persistent, split-K / stream-K over taps.
//
// Why fp16 pairs instead of tf32 pairs: the kernel is bound by bytes moved into shared memory (LDGSTS issue rate for the
// row gathers, L2->SM bandwidth for the weight slices), not by the tensor pipe.  The fp16 pair x = hi + lo' * 2^-11
// (h16.cuh) carries the same 22 mantissa bits as the tf32 pair in HALF the bytes: a split row is as large as the plain
// fp32 row, a 32-channel slice of a row is one 128-byte line holding both halves, fp16 wgmma run at twice the tf32 rate,
// and the weight image halves too.  Range: |x| < 65504 (flagged in `status` bit 0 otherwise); the tf32-pair kernel
// (sparse_conv_tc.cu) stays available for data outside that range.
//
//   D[0, N)    += A_hi  x B_hi                      (N = Cout)
//   D[N, 2N)   += A_hi  x B_lo' + A_lo' x B_hi      (both scaled by 2^11)         out = D[0,N) + D[N,2N) * 2^-11
//   -> per 16-channel k-step three m64nN wgmma per warpgroup; the weight k-block holds [B_hi | B_lo'] as 2N K-major rows.
//
// Row layout H16 of a C-channel row (4*C bytes): groups of KC = min(C, 32) channels, each [hi KC halfs | lo' KC halfs].
// Shared-memory operand "sub-tile": 128 rows x 128 bytes, SWIZZLE_128B K-major (64 fp16 = 4 k-steps of 16):
//   C >= 32: one (tap, 32-channel group): k-steps 0,1 = hi, 2,3 = lo'  -> one 128-byte line per gathered row
//   C == 16: two taps: k-steps 0,1 = hi, lo' of tap a; 2,3 = hi, lo' of tap b -> two 64-byte half lines per row
// A pipeline stage = NSUB sub-tiles + their weight blocks (NSUB = 2 for Cin <= 32 and Cout <= 64, else 1).
//
// CTA = 1 per SM, two warpgroups (warpgroup g: rows 64g .. 64g+63 of the 128-row tile), persistent over work items (tile
// of 128 output rows, tap split).  Every thread gathers rows with cp.async (zero-fill for missing neighbours) STAGES - 1
// stages ahead of the tensor cores, thread 0 copies the weight blocks with cp.async.bulk (mbarrier complete_tx); after
// the last stage the warpgroups run the epilogue (split-K fix-up, BN / bias / residual / ReLU, fp32 and / or H16 rows)
// straight from their accumulator fragments.
// Split-K / stream-K over taps (few tiles on the deep levels): the decomposition (no split, 2-4 tap splits or stream-K)
// is chosen ON THE DEVICE from the row count so that the work items fill the grid; partial tiles go to scratch slabs and
// the LAST arriving CTA of a tile (ticket counter) sums the slabs in index order (deterministic) and runs the fused
// epilogue - no finalize launch.  Nothing else runs on the SM during an epilogue, so its global loads (slabs, residual
// rows) are issued a fragment at a time, not one dependent round trip per pair.  Launched with PDL (launch_pdl).
#include <cuda.h>
#include <cuda_fp16.h>

#include "h16.cuh"
#include "tc_common.cuh"

namespace p3d {
namespace f16 {

using namespace tc;

constexpr int kSub = 128 * 128;  // bytes of one A sub-tile
constexpr int kMaxSplits = 4;
constexpr int kMaxStages = 12;
constexpr int kSkFix = 6;  // cost of a stream-K tile's fix-up (slab writes, ticket, slab sums) in taps

template <int CIN, int COUT>
struct Cfg {
  static constexpr int KC = (CIN >= 32) ? 32 : 16;
  static constexpr int G = CIN / KC;                         // sub-tiles per tap (CIN >= 32); CIN == 16: 2 taps / sub-tile
  static constexpr int NSUB = (CIN <= 32 && COUT <= 64) ? 2 : 1;  // sub-tiles per stage: 4 (Cin 16) / 2 (Cin 32) taps
  static constexpr int B_SUB = 128 * COUT;                   // bytes of the weight blocks of one sub-tile (2 k-blocks)
  static constexpr int B_BLK = 64 * COUT;                    // one 16-channel k-block: [2 chunks][2*COUT rows][16 B]
  static constexpr int STAGE = NSUB * (kSub + B_SUB);
  // ring depth from the shared-memory budget: 227 KB - 1 KB alignment slack - 16 KB neighbour map (K <= 32) - 3 KB static
  static constexpr int BUDGET = (227 - 1 - 16 - 3) * 1024;
  static constexpr int S_RAW = BUDGET / STAGE;
  static constexpr int STAGES = S_RAW > kMaxStages ? kMaxStages : S_RAW;
  static constexpr int ACC = COUT;  // fp32 registers per thread: m64 x 2*COUT per warpgroup
  static_assert(CIN % 16 == 0 && COUT % 16 == 0 && COUT <= 128 && CIN <= 128, "16-channel multiples up to 128");
  static_assert(CIN == 16 || CIN % 32 == 0, "CIN = 16 or a multiple of 32");
  static_assert(STAGE % 1024 == 0, "SWIZZLE_128B tiles need 1024-byte alignment");
  static_assert(STAGES >= 3, "ring too shallow");
};

// Number of tap splits for `n_tiles` row tiles on `grid` persistent CTAs: minimise waves x (taps per item + fixed cost).
__host__ __device__ inline int choose_splits(long long n_tiles, int grid, int K, int smax) {
  if (smax > K) smax = K;
  if (smax < 1) smax = 1;
  int best = 1;
  long long best_cost = -1;
  for (int s = 1; s <= smax; ++s) {
    const long long waves = (n_tiles * s + grid - 1) / grid;
    const long long cost = waves * ((K + s - 1) / s + 4 + (s > 1 ? 1 : 0));
    if (best_cost < 0 || cost < best_cost) {
      best_cost = cost;
      best = s;
    }
  }
  return best;
}
// taps of split `split` (t == split mod splits), K <= 32
__device__ __forceinline__ uint32_t split_taps(int split, int splits, int K) {
  uint32_t m = 0u;
  for (int t = split; t < K; t += splits) m |= 1u << t;
  return m;
}

// Work decomposition of one launch.  stream = 0: items (tile, split), split s owns the taps t == s (mod splits), item
// w = blockIdx.x + it * gridDim.x.  stream = 1 ("stream-K"): the n_tiles * K (tile, tap) units are cut into g_eff equal
// contiguous ranges, one per CTA; a CTA's items are the tiles its range touches, each with the contiguous tap range that
// falls inside.  A tile cut by range boundaries has `pieces` partial sums (its CTAs are consecutive: piece = CTA - first
// CTA), combined through the slabs / ticket like the splits.  No wave quantisation: e.g. 309 tiles on 132 CTAs cost 64 taps
// per CTA instead of 3 x 27.  Ranges are never shorter than ceil((K - 1) / (kMaxSplits - 1)) units, so pieces <= kMaxSplits.
// Stream-K needs slabs for kMaxSplits pieces and runs when its cost (taps per CTA + kSkFix) beats the split schedule's.
struct Sched {
  int stream, splits, K;
  long long n_work;          // stream = 0: n_tiles * splits
  long long total, g_eff;    // stream = 1
  long long u0, u1;          // stream = 1: this CTA's unit range
};
__device__ __forceinline__ Sched make_sched(long long n_tiles, int K, int smax) {
  Sched sc;
  sc.K = K;
  sc.stream = 0;
  const int grid = static_cast<int>(gridDim.x);
  sc.splits = choose_splits(n_tiles, grid, K, smax);
  sc.n_work = n_tiles * sc.splits;
  sc.total = n_tiles * K;
  sc.g_eff = 1;
  sc.u0 = sc.u1 = 0;
  if (smax >= 4 && sc.total > 0) {  // slabs for 4 pieces available
    const int u_min = (K - 1 + 2) / 3 > 1 ? (K - 1 + 2) / 3 : 1;  // ceil((K - 1) / (kMaxSplits - 1)), kMaxSplits = 4
    long long g = sc.total / u_min;
    if (g > grid) g = grid;
    if (g < 1) g = 1;
    const long long waves = (sc.n_work + grid - 1) / grid;
    const long long cost_old = waves * ((K + sc.splits - 1) / sc.splits + 4 + (sc.splits > 1 ? 1 : 0));
    const long long cost_stream = (sc.total + g - 1) / g + 4 + kSkFix;
    if (cost_stream < cost_old) {
      sc.stream = 1;
      sc.g_eff = g;
      const long long c = blockIdx.x;
      if (c < g) {
        sc.u0 = c * sc.total / g;
        sc.u1 = (c + 1) * sc.total / g;
      }
    }
  }
  return sc;
}
// item `it` of this CTA: false when the CTA has no more items
__device__ __forceinline__ bool sched_item(const Sched &sc, int it, long long &tile, uint32_t &mask, int &piece, int &pieces) {
  if (!sc.stream) {
    const long long w = static_cast<long long>(blockIdx.x) + static_cast<long long>(it) * gridDim.x;
    if (w >= sc.n_work) return false;
    tile = w / sc.splits;
    piece = static_cast<int>(w - tile * sc.splits);
    pieces = sc.splits;
    mask = split_taps(piece, pieces, sc.K);
    return true;
  }
  tile = sc.u0 / sc.K + it;
  const long long start = tile * sc.K;
  if (start >= sc.u1) return false;
  const int ta = static_cast<int>((sc.u0 > start ? sc.u0 : start) - start);
  const int tb = static_cast<int>((sc.u1 < start + sc.K ? sc.u1 : start + sc.K) - start);
  mask = (tb >= 32 ? 0xffffffffu : ((1u << tb) - 1u)) & ~((1u << ta) - 1u);
  const long long cf = ((start + 1) * sc.g_eff - 1) / sc.total, cl = ((start + sc.K) * sc.g_eff - 1) / sc.total;
  piece = static_cast<int>(static_cast<long long>(blockIdx.x) - cf);
  pieces = static_cast<int>(cl - cf + 1);
  return true;
}

struct Params {
  const uint8_t *in;        // H16 rows [n_in][4 * CIN bytes]
  const int32_t *nbr;       // [n_cap][K]
  const int32_t *n_out_dev; // device row count (or null: n_cap)
  long long n_cap;
  int K;
  int smax;                 // max tap splits the workspace allows (1 = never split)
  const uint8_t *packed_w;  // [K * CIN / 16] k-blocks of 64 * COUT bytes
  const float *scale, *shift;
  const uint8_t *residual;  // H16 rows [n][4 * COUT bytes] or null
  int relu;
  float *out_f32;           // [n][COUT] or null
  uint8_t *out_h16;         // [n][4 * COUT bytes] or null
  float *slabs;             // split-K scratch [smax][tiles][128 rows][COUT] fp32 (smax > 1)
  int32_t *counters;        // split-K tickets [tiles], zero on entry, left zero
  int32_t *status;          // optional: bit 0 = fp16 range overflow while producing out_h16
};
__device__ __forceinline__ int nth_bit(uint32_t m, int k) {  // position of the k-th (0-based) set bit of m
  for (int i = 0; i < k; ++i) m &= m - 1u;
  return __ffs(m) - 1;
}

template <int CIN, int COUT>
__global__ void __launch_bounds__(kThreads, 1) conv_f16_kernel(const Params p) {
  using C = Cfg<CIN, COUT>;
  constexpr int S = C::STAGES, NSUB = C::NSUB;
  constexpr int H = COUT / 2;  // accumulator registers of the hi products; the cross products follow
  pdl_trigger();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) unsigned long long s_bar[kMaxStages + 1];    // full[S] (weight bytes) | neighbour map landed
  constexpr int kF = 0, kNR = kMaxStages;
  __shared__ int s_last;
  __shared__ float s_scale[COUT], s_shift[COUT];

  // barrier init and the BN constants read nothing the previous kernel wrote: they overlap its tail
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127;
  if (tid < COUT) {
    s_scale[tid] = p.scale ? __ldg(p.scale + tid) : 1.0f;
    s_shift[tid] = p.shift ? __ldg(p.shift + tid) : 0.0f;
  }
  if (tid == 0) {
    for (int s = 0; s < S; ++s) mbar_init(smem_u32(&s_bar[kF + s]), 1);
    mbar_init(smem_u32(&s_bar[kNR]), 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // the row count and the input rows are earlier kernels' output
  const long long n = p.n_out_dev ? min(static_cast<long long>(p.n_out_dev[0]), p.n_cap) : p.n_cap;
  const long long n_tiles = (n + kM - 1) / kM;
  const int K = p.K;
  const Sched sc = make_sched(n_tiles, K, p.smax);
  if (sc.stream ? (sc.u0 >= sc.u1) : (static_cast<long long>(blockIdx.x) >= sc.n_work)) return;
  int32_t *s_nbr = reinterpret_cast<int32_t *>(smem + S * C::STAGE);  // [kM * K]
  const uint32_t ring = smem_u32(smem);
  const int sub4 = tid >> 3, ch = tid & 7;  // gather: 32 rows x 8 16-byte chunks per CTA instruction
  constexpr int KCO = (COUT >= 32) ? 32 : 16;  // channels per H16 group of the output / residual rows
  const size_t tiles_cap = static_cast<size_t>((p.n_cap + kM - 1) / kM);
  bool ovf = false;
  uint32_t gu = 0;  // stages consumed by earlier items: the ring phases keep running

  // Every item's taps are known arithmetically (all K, or the split's / stream-K range's taps): a tap without any
  // neighbour in the tile just multiplies zero rows (rare: the rows of a tile are not spatially sorted), so nothing on
  // the critical path scans the map.
  long long tile;
  uint32_t m;
  int piece, pieces;
  for (int it = 0; sched_item(sc, it, tile, m, piece, pieces); ++it) {
    const long long row0 = tile * kM;
    const int rows = static_cast<int>(min(static_cast<long long>(kM), n - row0));
    const int n_taps = __popc(m);
    const int n_sub = (CIN == 16) ? (n_taps + 1) / 2 : n_taps * C::G;
    const int n_st = (n_sub + NSUB - 1) / NSUB;
    __syncthreads();  // previous item drained: s_nbr free
    {
      // the tile's neighbour map is one contiguous block of the [n_cap, K] array: one bulk copy; rows >= `rows` of the
      // block are never used
      const int avail = static_cast<int>(min(static_cast<long long>(kM), p.n_cap - row0));
      const uint32_t words = static_cast<uint32_t>(avail) * K, bulk_words = words & ~3u;
      if (tid == 0) {
        fence_proxy_async();  // earlier generic reads of s_nbr vs the async-proxy write
        mbar_arrive_expect_tx(smem_u32(&s_bar[kNR]), bulk_words * 4);
        if (bulk_words) bulk_g2s(smem_u32(s_nbr), p.nbr + row0 * K, bulk_words * 4, smem_u32(&s_bar[kNR]));
      }
      if (bulk_words + tid < words) s_nbr[bulk_words + tid] = __ldg(p.nbr + row0 * K + bulk_words + tid);  // <= 3 tail words
      __syncthreads();
      mbar_wait(smem_u32(&s_bar[kNR]), static_cast<uint32_t>(it & 1));
    }
    // stage q of this item: sub-tiles q * NSUB .. (rows gathered by every thread, weight blocks by thread 0)
    auto issue = [&](int q) {
      if (q >= n_st) return;
      const uint32_t slot = (gu + static_cast<uint32_t>(q)) % S;
      const uint32_t st = ring + slot * C::STAGE, bar = smem_u32(&s_bar[kF + slot]);
      const int k0 = q * NSUB, subs = min(NSUB, n_sub - k0);
      if (tid == 0) {
        const int bytes = (CIN == 16) ? min(2 * subs, n_taps - 2 * k0) * C::B_BLK : subs * C::B_SUB;
        mbar_arrive_expect_tx(bar, static_cast<uint32_t>(bytes));
      }
#pragma unroll
      for (int j = 0; j < NSUB; ++j) {
        const int k = k0 + j;
        if (k >= n_sub) break;
        const uint32_t sb = st + static_cast<uint32_t>(j * kSub);
        const uint32_t bb = st + static_cast<uint32_t>(NSUB * kSub + j * C::B_SUB);
        if (CIN == 16) {
          // threads 0-3 of a row fetch tap a's 64-byte row, 4-7 tap b's
          const int ta = nth_bit(m, 2 * k), tb = (2 * k + 1 < n_taps) ? nth_bit(m, 2 * k + 1) : -1;
          if (tid == 0) {
            bulk_g2s(bb, p.packed_w + static_cast<size_t>(ta) * C::B_BLK, C::B_BLK, bar);
            if (tb >= 0) bulk_g2s(bb + C::B_BLK, p.packed_w + static_cast<size_t>(tb) * C::B_BLK, C::B_BLK, bar);
          }
          const int t = (ch < 4) ? ta : tb;
          if (t >= 0) {
#pragma unroll
            for (int q4 = 0; q4 < 4; ++q4) {
              const int row = q4 * 32 + sub4;
              const int idx = row < rows ? s_nbr[row * K + t] : -1;
              const bool ok = idx >= 0;
              const uint8_t *src = p.in + static_cast<size_t>(max(idx, 0)) * 64 + (ch & 3) * 16;
              cp_async16(sb + static_cast<uint32_t>(row * 128 + ((ch ^ (row & 7)) << 4)), src, ok);
            }
          }
        } else {
          const int t = nth_bit(m, k / C::G), g = k % C::G;
          if (tid == 0) bulk_g2s(bb, p.packed_w + (static_cast<size_t>(t) * (CIN / 16) + 2 * g) * C::B_BLK, C::B_SUB, bar);
#pragma unroll
          for (int q4 = 0; q4 < 4; ++q4) {
            const int row = q4 * 32 + sub4;
            const int idx = row < rows ? s_nbr[row * K + t] : -1;
            const bool ok = idx >= 0;
            const uint8_t *src = p.in + static_cast<size_t>(max(idx, 0)) * (4 * CIN) + g * 128 + ch * 16;
            cp_async16(sb + static_cast<uint32_t>(row * 128 + ((ch ^ (row & 7)) << 4)), src, ok);
          }
        }
      }
    };

    float acc[C::ACC];
#pragma unroll
    for (int i = 0; i < C::ACC; ++i) acc[i] = 0.f;
    for (int q = 0; q < S - 1; ++q) {
      issue(q);
      cp_async_commit();
    }
    for (int q = 0; q < n_st; ++q) {
      const uint32_t slot = (gu + static_cast<uint32_t>(q)) % S, par = ((gu + static_cast<uint32_t>(q)) / S) & 1u;
      cp_async_wait<S - 2>();  // this thread's gathers of stage q have landed
      fence_proxy_async();     // cp.async (generic proxy) writes -> wgmma (async proxy) reads
      mbar_wait(smem_u32(&s_bar[kF + slot]), par);
      __syncthreads();         // whole stage present; the wgmma of stage q - 1 have retired in both warpgroups
      const uint32_t st = ring + slot * C::STAGE;
      wg_fence();
#pragma unroll
      for (int j = 0; j < NSUB; ++j) {
        const int k = q * NSUB + j;
        if (k < n_sub) {
          const uint32_t a_base = st + static_cast<uint32_t>(j * kSub + wg * 64 * 128);
          const uint32_t b_base = st + static_cast<uint32_t>(NSUB * kSub + j * C::B_SUB);
          const bool half_only = (CIN == 16) && (k == n_sub - 1) && (n_taps & 1);
#pragma unroll
          for (int kb = 0; kb < 2; ++kb) {
            if (kb == 1 && half_only) continue;
            const int ks_hi = (CIN == 16) ? 2 * kb : kb, ks_lo = (CIN == 16) ? 2 * kb + 1 : 2 + kb;
            const uint32_t bk = b_base + static_cast<uint32_t>(kb * C::B_BLK);
            const uint64_t dbh = smem_desc(bk, 2 * COUT * 16, 128), dbl = smem_desc(bk + COUT * 16, 2 * COUT * 16, 128);
            const uint64_t dah = desc_sw128(a_base + ks_hi * 32), dal = desc_sw128(a_base + ks_lo * 32);
            wg::mma_f16<COUT>(acc, dah, dbh, 1u);      // A_hi x B_hi
            wg::mma_f16<COUT>(acc + H, dah, dbl, 1u);  // A_hi x B_lo'
            wg::mma_f16<COUT>(acc + H, dal, dbh, 1u);  // A_lo' x B_hi
          }
        }
      }
      wg_commit();
      issue(q + S - 1);  // the slot of stage q - 1
      cp_async_commit();
      wg_wait<0>();
    }
    wg_fence_acc<C::ACC>(acc);
    cp_async_wait<0>();
    gu += static_cast<uint32_t>(n_st);

    // ------------------------------------------------------------------------------------------ epilogue
    // acc[i] (i < H) becomes the value of output column frag_col(i): hi products + cross products * 2^-11
#pragma unroll
    for (int i = 0; i < H; ++i) acc[i] = fmaf(acc[i + H], kLoInv, acc[i]);
    bool finish = true;  // this CTA runs the fused epilogue of the tile
    if (pieces > 1) {
      // split-K slabs [piece][tile][128 rows][COUT] fp32; rows beyond `rows` land in the slab's padding
      float *mine = p.slabs + ((static_cast<size_t>(piece) * tiles_cap + static_cast<size_t>(tile)) * kM) * COUT;
#pragma unroll
      for (int i = 0; i < H; i += 2) {
        const int r = wg * 64 + frag_row(i, wtid), c = frag_col(i, wtid);
        __stcg(reinterpret_cast<float2 *>(mine + r * COUT + c), make_float2(acc[i], acc[i + 1]));
      }
      __threadfence();
      __syncthreads();
      if (tid == 0) {
        const int old = atomicAdd(p.counters + tile, 1);
        const int last = (old == pieces - 1) ? 1 : 0;
        if (last) p.counters[tile] = 0;  // all pieces have arrived: leave the ticket clean for the next launch
        s_last = last;
      }
      __syncthreads();
      finish = s_last != 0;
      if (finish) {
        __threadfence();
        // slabs in index order (deterministic); slab outermost, so that a slab's loads are all in flight together
        // instead of one round trip per fragment pair
#pragma unroll
        for (int i = 0; i < H; ++i) acc[i] = 0.f;
        for (int sp = 0; sp < pieces; ++sp) {
          const float *slab = p.slabs + ((static_cast<size_t>(sp) * tiles_cap + static_cast<size_t>(tile)) * kM) * COUT;
          float2 t2[H / 2];
#pragma unroll
          for (int i = 0; i < H; i += 2) {
            const int r = wg * 64 + frag_row(i, wtid), c = frag_col(i, wtid);
            t2[i / 2] = __ldcg(reinterpret_cast<const float2 *>(slab + r * COUT + c));
          }
#pragma unroll
          for (int i = 0; i < H; i += 2) {
            acc[i] += t2[i / 2].x;
            acc[i + 1] += t2[i / 2].y;
          }
        }
      }
    }
    if (finish) {
      // the residual pairs of the whole fragment are loaded before the first output store (the compiler cannot move a
      // load above a store that may alias it): one round trip instead of one per fragment pair
      __half2 rhi[H / 2], rlo[H / 2];
      if (p.residual) {
#pragma unroll
        for (int i = 0; i < H; i += 2) {
          const int r = wg * 64 + frag_row(i, wtid), c = frag_col(i, wtid);
          if (r >= rows) continue;
          const uint8_t *rp = p.residual + static_cast<size_t>(row0 + r) * (4 * COUT) + (c / KCO) * (4 * KCO) + (c % KCO) * 2;
          rhi[i / 2] = *reinterpret_cast<const __half2 *>(rp);
          rlo[i / 2] = *reinterpret_cast<const __half2 *>(rp + 2 * KCO);
        }
      }
#pragma unroll
      for (int i = 0; i < H; i += 2) {
        const int r = wg * 64 + frag_row(i, wtid), c = frag_col(i, wtid);
        if (r >= rows) continue;
        const size_t orow = static_cast<size_t>(row0 + r);
        const size_t goff = static_cast<size_t>((c / KCO) * (4 * KCO) + (c % KCO) * 2);  // byte offset of the hi pair
        float v[2] = {acc[i], acc[i + 1]};
        float res[2] = {0.f, 0.f};
        if (p.residual) {
          const __half2 hh = rhi[i / 2], ll = rlo[i / 2];
          res[0] = merge_h16(__low2half(hh), __low2half(ll));
          res[1] = merge_h16(__high2half(hh), __high2half(ll));
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float o = fmaf(v[e], s_scale[c + e], s_shift[c + e]);
          if (p.residual) o = o + res[e];
          if (p.relu) o = fmaxf(o, 0.f);
          v[e] = o;
        }
        if (p.out_f32) *reinterpret_cast<float2 *>(p.out_f32 + orow * COUT + c) = make_float2(v[0], v[1]);
        if (p.out_h16) {
          __half h0, l0, h1, l1;
          split_h16(v[0], h0, l0, ovf);
          split_h16(v[1], h1, l1, ovf);
          uint8_t *op = p.out_h16 + orow * (4 * COUT) + goff;
          *reinterpret_cast<__half2 *>(op) = __halves2half2(h0, h1);
          *reinterpret_cast<__half2 *>(op + 2 * KCO) = __halves2half2(l0, l1);
        }
      }
    }
  }
  if (ovf && p.status) atomicOr(p.status, 1);
}

template <int CIN, int COUT>
int launch(const Params &p, cudaStream_t st) {
  using C = Cfg<CIN, COUT>;
  const size_t smem = static_cast<size_t>(C::STAGES) * C::STAGE + static_cast<size_t>(kM) * p.K * sizeof(int32_t) + 1024;
  if (smem > 227 * 1024) return P3D_ERR_UNSUPPORTED;
  auto kern = conv_f16_kernel<CIN, COUT>;
  P3D_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  const long long work = ((p.n_cap + kM - 1) / kM) * (p.smax > 1 ? p.smax : 1);
  const long long sms = num_sms();
  const unsigned int grid = static_cast<unsigned int>(work < sms ? work : sms);
  P3D_CUDA_CHECK(launch_pdl(kern, dim3(grid), dim3(kThreads), smem, st, p));
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

// fp32 [K][Cin][Cout] -> k-blocks [K * Cin / 16][2 chunks][2 * Cout rows (hi, then lo')][8 halfs]
__global__ void __launch_bounds__(256) pack_weights_kernel(const float *__restrict__ w, int K, int Cin, int Cout,
                                                           __half *__restrict__ packed, int32_t *status) {
  const long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(K) * Cin * Cout;
  if (q >= total) return;
  const int n = static_cast<int>(q % Cout);
  const int ci = static_cast<int>((q / Cout) % Cin);
  const int t = static_cast<int>(q / (static_cast<long long>(Cout) * Cin));
  const size_t kb = static_cast<size_t>(t) * (Cin / 16) + ci / 16;
  const int c = (ci % 16) / 8, j = ci % 8;
  __half hi, lo;
  bool ovf = false;
  split_h16(w[q], hi, lo, ovf);
  const size_t blk = kb * static_cast<size_t>(32 * Cout);  // halfs per k-block = 64 * Cout / 2
  packed[blk + (static_cast<size_t>(c) * (2 * Cout) + n) * 8 + j] = hi;
  packed[blk + (static_cast<size_t>(c) * (2 * Cout) + Cout + n) * 8 + j] = lo;
  if (ovf && status) atomicOr(status, 1);
}

// rows [n, C] fp32 <-> H16 rows
__global__ void __launch_bounds__(256) rows_to_h16_kernel(const float *__restrict__ x, const int32_t *__restrict__ n_dev,
                                                          long long n_cap, int C, __half *__restrict__ out, int32_t *status) {
  const long long n = n_dev ? min(static_cast<long long>(n_dev[0]), n_cap) : n_cap;
  const long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (q >= n * C) return;
  const long long r = q / C;
  const int c = static_cast<int>(q - r * C);
  const int KC = C >= 32 ? 32 : 16;
  __half hi, lo;
  bool ovf = false;
  split_h16(x[q], hi, lo, ovf);
  __half *row = out + r * 2 * C + (c / KC) * (2 * KC);
  row[c % KC] = hi;
  row[KC + c % KC] = lo;
  if (ovf && status) atomicOr(status, 1);
}
__global__ void __launch_bounds__(256) rows_from_h16_kernel(const __half *__restrict__ xs, const int32_t *__restrict__ n_dev,
                                                            long long n_cap, int C, float *__restrict__ out) {
  const long long n = n_dev ? min(static_cast<long long>(n_dev[0]), n_cap) : n_cap;
  const long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (q >= n * C) return;
  const long long r = q / C;
  const int c = static_cast<int>(q - r * C);
  const int KC = C >= 32 ? 32 : 16;
  const __half *row = xs + r * 2 * C + (c / KC) * (2 * KC);
  out[q] = merge_h16(row[c % KC], row[KC + c % KC]);
}

}  // namespace f16
}  // namespace p3d

using namespace p3d;

extern "C" size_t p3d_sparse_conv_f16_packed_weight_bytes(int K, int Cin, int Cout) {
  if (K < 1 || K > 32 || Cin < 16 || Cout < 16 || Cin > 128 || Cout > 128 || Cout % 16 || (Cin != 16 && Cin % 32)) return 0;
  return align_up(static_cast<size_t>(K) * Cin * Cout * 4);
}

extern "C" int p3d_sparse_conv_f16_pack_weights(const float *weight, int K, int Cin, int Cout, void *packed,
                                                int32_t *status_dev, p3d_stream_t stream) {
  if (!weight || !packed || K < 1) return P3D_ERR_INVALID_ARG;
  if (!p3d_sparse_conv_f16_packed_weight_bytes(K, Cin, Cout)) return P3D_ERR_UNSUPPORTED;
  const long long total = static_cast<long long>(K) * Cin * Cout;
  f16::pack_weights_kernel<<<div_up(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      weight, K, Cin, Cout, static_cast<__half *>(packed), status_dev);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

// dense layers (csrc/dense_conv_f16.cu): the same k-block image for one N tile, W[tap][Cin][n_tile], any Cin % 32 == 0
extern "C" int p3d_dense_conv2d_f16_pack_weights(const float *weight_tci, int taps, int Cin, int n_tile, void *packed,
                                                 int32_t *status_dev, p3d_stream_t stream) {
  if (!weight_tci || !packed || taps < 1 || Cin < 32 || Cin % 32 || (n_tile != 16 && n_tile != 32 && n_tile != 64 && n_tile != 128))
    return P3D_ERR_INVALID_ARG;
  const long long total = static_cast<long long>(taps) * Cin * n_tile;
  f16::pack_weights_kernel<<<div_up(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      weight_tci, taps, Cin, n_tile, static_cast<__half *>(packed), status_dev);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" int p3d_rows_convert_h16(const void *src, int to_h16, const int32_t *n_dev, int64_t n_cap, int C, void *dst,
                                    int32_t *status_dev, p3d_stream_t stream) {
  if (n_cap < 0 || C < 16 || (C != 16 && C % 32) || (n_cap && (!src || !dst))) return P3D_ERR_INVALID_ARG;
  if (n_cap == 0) return P3D_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (to_h16)
    f16::rows_to_h16_kernel<<<div_up(n_cap * C, 256), 256, 0, st>>>(static_cast<const float *>(src), n_dev, n_cap, C,
                                                                    static_cast<__half *>(dst), status_dev);
  else
    f16::rows_from_h16_kernel<<<div_up(n_cap * C, 256), 256, 0, st>>>(static_cast<const __half *>(src), n_dev, n_cap, C,
                                                                      static_cast<float *>(dst));
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

// workspace = [tickets: one int32 per 128-row tile][slabs: max_splits x n_out_cap x Cout fp32]; 0 for max_splits <= 1
extern "C" size_t p3d_sparse_conv_f16_workspace_bytes(int64_t n_out_cap, int Cout, int max_splits) {
  if (n_out_cap <= 0 || Cout < 16 || max_splits <= 1) return 0;
  if (max_splits > f16::kMaxSplits) max_splits = f16::kMaxSplits;
  const size_t tiles = static_cast<size_t>((n_out_cap + tc::kM - 1) / tc::kM);
  return align_up(tiles * sizeof(int32_t)) + align_up(static_cast<size_t>(max_splits) * tiles * tc::kM * Cout * sizeof(float));
}

extern "C" int p3d_sparse_conv_f16(const void *in_h16, const int32_t *nbr, const int32_t *n_out_dev, int64_t n_out_cap,
                                   int K, int Cin, int Cout, const void *packed_weight, const float *scale,
                                   const float *shift, const void *residual_h16, int relu, float *out_f32, void *out_h16,
                                   void *workspace, size_t workspace_bytes, int max_splits, int32_t *status_dev,
                                   p3d_stream_t stream) {
  if (n_out_cap < 0 || K < 1 || K > 32 || !packed_weight || (!out_f32 && !out_h16) || (n_out_cap && (!in_h16 || !nbr)))
    return P3D_ERR_INVALID_ARG;
  if (n_out_cap == 0) return P3D_OK;
  if ((reinterpret_cast<uintptr_t>(in_h16) & 15) || (reinterpret_cast<uintptr_t>(out_f32) & 15) ||
      (reinterpret_cast<uintptr_t>(out_h16) & 15) || (reinterpret_cast<uintptr_t>(packed_weight) & 15) ||
      (reinterpret_cast<uintptr_t>(residual_h16) & 15) || (reinterpret_cast<uintptr_t>(workspace) & 15) ||
      (reinterpret_cast<uintptr_t>(nbr) & 15))
    return P3D_ERR_INVALID_ARG;
  f16::Params p;
  p.in = static_cast<const uint8_t *>(in_h16);
  p.nbr = nbr;
  p.n_out_dev = n_out_dev;
  p.n_cap = n_out_cap;
  p.K = K;
  p.packed_w = static_cast<const uint8_t *>(packed_weight);
  p.scale = scale;
  p.shift = shift;
  p.residual = static_cast<const uint8_t *>(residual_h16);
  p.relu = relu;
  p.out_f32 = out_f32;
  p.out_h16 = static_cast<uint8_t *>(out_h16);
  p.status = status_dev;
  // split-K is available up to the number of slabs the workspace holds
  int smax = max_splits;
  if (smax > f16::kMaxSplits) smax = f16::kMaxSplits;
  if (smax > K) smax = K;
  const size_t tiles = static_cast<size_t>((n_out_cap + tc::kM - 1) / tc::kM);
  const size_t tick = align_up(tiles * sizeof(int32_t));
  const size_t slab = tiles * tc::kM * static_cast<size_t>(Cout) * sizeof(float);  // whole tiles: [tile][128 rows][Cout]
  if (!workspace || workspace_bytes < tick + 2 * slab) smax = 1;
  if (smax > 1) {
    const size_t fit = (workspace_bytes - tick) / slab;
    if (static_cast<size_t>(smax) > fit) smax = static_cast<int>(fit);
  }
  p.smax = smax < 1 ? 1 : smax;
  p.counters = p.smax > 1 ? static_cast<int32_t *>(workspace) : nullptr;
  p.slabs = p.smax > 1 ? reinterpret_cast<float *>(static_cast<char *>(workspace) + tick) : nullptr;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (Cin == 16 && Cout == 16) return f16::launch<16, 16>(p, st);
  if (Cin == 16 && Cout == 32) return f16::launch<16, 32>(p, st);
  if (Cin == 32 && Cout == 32) return f16::launch<32, 32>(p, st);
  if (Cin == 32 && Cout == 64) return f16::launch<32, 64>(p, st);
  if (Cin == 64 && Cout == 64) return f16::launch<64, 64>(p, st);
  if (Cin == 64 && Cout == 128) return f16::launch<64, 128>(p, st);
  if (Cin == 128 && Cout == 128) return f16::launch<128, 128>(p, st);
  return P3D_ERR_UNSUPPORTED;
}
