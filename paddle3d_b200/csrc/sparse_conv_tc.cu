// Sparse-conv gather-GEMM on Hopper tensor cores, 3xTF32: wgmma kind tf32 with fp32 accumulators in registers; every
// operand is split into tf32 hi + lo (D += a_hi*b_hi + a_hi*b_lo + a_lo*b_hi) for fp32-level accuracy.  This is the
// fallback of the fp16-pair kernels for activations outside fp16's range.
//
// One kernel serves two row layouts of the activations (template argument SPLIT_ROWS):
//   fp32 rows [n][C]       the gather loads a row into registers and splits it there, once per gathering neighbour;
//                          residual and output are fp32 rows.
//   split rows [n][2][C]   tf32 hi row, then lo row, split ONCE per element in the producing layer's epilogue; the gather
//                          is a pure cp.async copy (16 B, zero-fill for a missing neighbour) into the operand tiles.  The
//                          residual is split rows; the output fp32 rows, split rows for the next layer, or both.
// Both fill the same swizzled hi / lo tiles and run the same wgmma sequence, so equal values give equal bits.
//
//   grid        persistent: min(#work items at capacity, MIN_CTAS x SMs) CTAs, each walks the work items
//               w = blockIdx.x, +gridDim.x, ... (w = tile * splits + split) of the DEVICE row count.
//   CTA         two warpgroups; warpgroup g owns rows 64g .. 64g+63 of the 128-row tile (one m64nCout accumulator).
//   gather      the tile's neighbour map arrives with one bulk copy; taps that no row of the tile uses are skipped.  Per
//               (tap, KC-channel chunk) "use", the rows go into SWIZZLE_128B (KC = 32) or SWIZZLE_64B (KC = 16) tiles,
//               STAGES - 1 uses ahead; thread 0 copies the packed [hi | lo] weight slice of the use with cp.async.bulk
//               (mbarrier complete_tx).
//   mma         3 wgmma kind tf32 per 8-wide k-step: lo x hi + hi x lo into one accumulator, hi x hi into a second one
//               (the small cross terms keep their own rounding; the epilogue adds the two).  The hi x hi accumulator
//               holds one tap's partial sum only: after a tap's last channel chunk it is added to an fp32 register
//               total with round-to-nearest FADDs.  The tensor core's own accumulation is not round-to-nearest, so one
//               chain of 27 x Cin / 8 k-steps drifts (H100, 128 -> 128, K = 27: 1.5e-4 relative at 1e-2 x max, against
//               1.4e-5 with the per-tap total); per tap, both row layouts still run the same sums.
//   epilogue    BN scale/shift (+bias), residual, ReLU from the accumulator fragment.
//   split-K     the wide layers (Cout >= 64) have few 128-row tiles (52 - 130 at the C3 sizes): given a workspace, their
//               taps are spread over 2 CTAs per tile (split s owns the taps t == s mod splits), which write raw partial
//               sums to slab s; rows_finalize_kernel adds the slabs in slab order (deterministic) and runs the epilogue.
#include "tc_common.cuh"

namespace p3d {
namespace tc {

template <int CIN, int COUT, bool SPLIT_ROWS>
struct Cfg {
  // One pipeline "use" = one tap x KC input channels for the CTA's 128 rows.  Split rows take 32 channels (one whole
  // 128-byte line per row half); fp32 rows take 16, which keeps their ring at 4 - 6 stages and, for Cout <= 64, two CTAs
  // per SM (32-channel stages would need 120 - 144 KB there).
  static constexpr int KC = (SPLIT_ROWS && CIN >= 32) ? 32 : 16;
  static constexpr int G = CIN / KC;
  static constexpr int CH = KC / 4;                      // 16-byte chunks of a row per use
  static constexpr int A_TILE = KC * kM * 4;             // one of hi / lo
  static constexpr int A_STAGE = 2 * A_TILE;
  static constexpr int B_STAGE = 2 * KC * COUT * 4;      // [chunk][hi rows | lo rows][16 B]
  static constexpr int STAGE = A_STAGE + B_STAGE;        // ONE ring: rows and weights of a use share a slot
  static constexpr int MIN_CTAS = COUT <= 64 ? 2 : 1;
  static constexpr int BUDGET = COUT <= 64 ? 96 * 1024 : 192 * 1024;
  static constexpr int S_RAW = BUDGET / STAGE;
  static constexpr int STAGES = S_RAW > 8 ? 8 : (S_RAW < 3 ? 3 : S_RAW);
  static constexpr int ACC = COUT / 2;                   // registers of one m64 x COUT accumulator per thread
  static_assert(CIN % 16 == 0 && COUT % 16 == 0 && COUT <= 128, "tensor-core path needs 16-channel multiples");
  static_assert(STAGE % 1024 == 0 || KC == 16, "SWIZZLE_128B tiles need 1024-byte alignment");
  static_assert(STAGE % 512 == 0, "SWIZZLE_64B tiles need 512-byte alignment");
};

// split-K factor: taps spread over this many CTAs per 128-row tile
constexpr int splits_for(int Cout) { return Cout >= 64 ? 2 : 1; }

__device__ __forceinline__ int nth_bit(uint32_t m, int k) {  // position of the k-th (0-based) set bit of m
  for (int i = 0; i < k; ++i) m &= m - 1u;
  return __ffs(m) - 1;
}

// byte offset of 16-byte chunk `ch` of row `row` in an A tile: SWIZZLE_128B (row pitch 128 B, chunk ^= row & 7) for
// KC = 32, SWIZZLE_64B (row pitch 64 B, chunk ^= (row >> 1) & 3) for KC = 16
template <int KC>
__device__ __forceinline__ uint32_t a_off(int row, int ch) {
  return KC == 32 ? static_cast<uint32_t>(row * 128 + ((ch ^ (row & 7)) << 4))
                  : static_cast<uint32_t>(row * 64 + ((ch ^ ((row >> 1) & 3)) << 4));
}

template <int CIN, int COUT, bool SPLIT_ROWS>
__global__ void __launch_bounds__(kThreads, Cfg<CIN, COUT, SPLIT_ROWS>::MIN_CTAS)
    gather_gemm_tf32_kernel(const float *__restrict__ in, const int32_t *__restrict__ nbr,
                            const int32_t *__restrict__ n_out_dev, long long n_cap, int K, int splits,
                            const float *__restrict__ packed_w, const float *__restrict__ scale,
                            const float *__restrict__ shift, const float *__restrict__ residual, int relu,
                            float *__restrict__ out_f32, float *__restrict__ out_split) {
  using C = Cfg<CIN, COUT, SPLIT_ROWS>;
  constexpr int S = C::STAGES;
  pdl_trigger();
  pdl_wait();  // inputs of the previous layer are complete
  const long long n = n_out_dev ? min(static_cast<long long>(n_out_dev[0]), n_cap) : n_cap;
  // with splits > 1 the caller passes the scratch slabs as out_f32 and no epilogue operands
  const long long n_work = ((n + kM - 1) / kM) * splits;
  if (static_cast<long long>(blockIdx.x) >= n_work) return;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  int32_t *s_nbr = reinterpret_cast<int32_t *>(smem + S * C::STAGE);  // [kM][K]
  __shared__ __align__(8) unsigned long long s_full[S];             // weights of a stage landed
  __shared__ __align__(8) unsigned long long s_nbr_full;            // neighbour map of the item landed
  __shared__ uint32_t s_active;                                      // bit t: some row uses tap t (K <= 32)

  const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7, wtid = tid & 127;
  if (tid == 0) {
    for (int s = 0; s < S; ++s) mbar_init(smem_u32(&s_full[s]), 1);
    mbar_init(smem_u32(&s_nbr_full), 1);
    fence_mbar_init();
  }
  __syncthreads();
  const uint32_t ring = smem_u32(smem);
  // the bulk copy needs a 16-byte aligned source; the fp32-row entry points accept any int32 neighbour map
  const bool nbr_bulk = (reinterpret_cast<uintptr_t>(nbr) & 15) == 0;

  uint32_t gu = 0;  // uses of earlier work items: the ring phases keep running
  int item_it = 0;
  for (long long w = blockIdx.x; w < n_work; w += gridDim.x, ++item_it) {
    const long long tile = w / splits;
    const int split = static_cast<int>(w - tile * splits);
    float *out_rows = out_f32 ? out_f32 + static_cast<size_t>(split) * static_cast<size_t>(n_cap) * COUT : nullptr;
    uint32_t tap_mask = 0xffffffffu;
    if (splits > 1) {
      tap_mask = 0u;
      for (int t = split; t < K; t += splits) tap_mask |= 1u << t;
    }
    const long long row0 = tile * kM;
    const int rows = static_cast<int>(min(static_cast<long long>(kM), n - row0));
    __syncthreads();  // previous item fully drained (s_nbr free)
    if (tid == 0) s_active = 0u;
    {
      // the tile's neighbour map is one contiguous block of the [n_cap, K] array: one bulk copy instead of a
      // latency-bound load loop; rows >= `rows` of the block are never used.
      const int avail = static_cast<int>(min(static_cast<long long>(kM), n_cap - row0));
      const uint32_t words = static_cast<uint32_t>(avail) * K, bulk_words = nbr_bulk ? words & ~3u : 0u;
      if (tid == 0) {
        fence_proxy_async();  // earlier generic reads of s_nbr vs the async-proxy write
        mbar_arrive_expect_tx(smem_u32(&s_nbr_full), bulk_words * 4);
        if (bulk_words) bulk_g2s(smem_u32(s_nbr), nbr + row0 * K, bulk_words * 4, smem_u32(&s_nbr_full));
      }
      for (uint32_t q = bulk_words + tid; q < words; q += kThreads) s_nbr[q] = __ldg(nbr + row0 * K + q);
      __syncthreads();  // s_active reset and the words outside the bulk copy are plain stores
      mbar_wait(smem_u32(&s_nbr_full), static_cast<uint32_t>(item_it & 1));
      uint32_t mine = 0u;
      for (int q = tid; q < rows * K; q += kThreads)
        if (s_nbr[q] >= 0) mine |= 1u << (q % K);
      mine = __reduce_or_sync(0xffffffffu, mine);
      if (lane == 0 && mine) atomicOr(&s_active, mine);
    }
    __syncthreads();
    const uint32_t active = s_active & tap_mask;
    const int n_uses = __popc(active) * C::G;

    // gather use q (tap, chunk) of this item into its ring slot; thread 0 posts the weight slice on the slot's barrier
    auto issue = [&](int q) {
      if (q >= n_uses) return;
      const int t = nth_bit(active, q / C::G), g = q % C::G;
      const uint32_t slot = (gu + static_cast<uint32_t>(q)) % S;
      const uint32_t st = ring + slot * C::STAGE, bar = smem_u32(&s_full[slot]);
      if (tid == 0) {
        mbar_arrive_expect_tx(bar, static_cast<uint32_t>(C::B_STAGE));
        bulk_g2s(st + C::A_STAGE, packed_w + (static_cast<size_t>(t) * CIN + g * C::KC) * (2 * COUT),
                 static_cast<uint32_t>(C::B_STAGE), bar);
      }
      if constexpr (SPLIT_ROWS) {
        const int sub = tid >> 3;  // 32 rows per CTA instruction
        if (C::KC == 32) {
          // the hi and the lo line of a row: 8 threads per line
          const int ch = tid & 7;
#pragma unroll
          for (int q4 = 0; q4 < 4; ++q4) {
            const int row = q4 * 32 + sub;
            const int src = row < rows ? s_nbr[row * K + t] : -1;
            const bool ok = src >= 0;
            const float *p = in + (ok ? static_cast<size_t>(src) * (2 * CIN) : 0) + g * 32 + ch * 4;
            const uint32_t d = st + a_off<C::KC>(row, ch);
            cp_async16(d, p, ok);                    // hi
            cp_async16(d + C::A_TILE, p + CIN, ok);  // lo
          }
        } else {
          // 16-channel layers: a split row [hi 16 | lo 16] is ONE line (threads 0-3 of a row fetch the hi chunks,
          // 4-7 the lo chunks)
          const int ch = tid & 3, part = (tid >> 2) & 1;
#pragma unroll
          for (int q4 = 0; q4 < 4; ++q4) {
            const int row = q4 * 32 + sub;
            const int src = row < rows ? s_nbr[row * K + t] : -1;
            const bool ok = src >= 0;
            const float *p = in + (ok ? static_cast<size_t>(src) * (2 * CIN) : 0) + part * CIN + g * 16 + ch * 4;
            cp_async16(st + part * C::A_TILE + a_off<C::KC>(row, ch), p, ok);
          }
        }
      } else {
        // two threads per row, CH / 2 chunks each: the 32 lanes of one store instruction write the same chunk of 32
        // consecutive rows, which the swizzle spreads over all banks
        const int row = tid & (kM - 1), c0 = (tid >> 7) * (C::CH / 2);
        const int src = row < rows ? s_nbr[row * K + t] : -1;
        float4 v[C::CH / 2];
#pragma unroll
        for (int c = 0; c < C::CH / 2; ++c)
          v[c] = src >= 0 ? __ldg(reinterpret_cast<const float4 *>(in + static_cast<size_t>(src) * CIN + g * C::KC) + c0 + c)
                          : make_float4(0.f, 0.f, 0.f, 0.f);
        uint8_t *tile_hi = smem + slot * C::STAGE;
#pragma unroll
        for (int c = 0; c < C::CH / 2; ++c) {
          float4 h, l;
          split_tf32(v[c].x, h.x, l.x);
          split_tf32(v[c].y, h.y, l.y);
          split_tf32(v[c].z, h.z, l.z);
          split_tf32(v[c].w, h.w, l.w);
          const uint32_t off = a_off<C::KC>(row, c0 + c);
          *reinterpret_cast<float4 *>(tile_hi + off) = h;
          *reinterpret_cast<float4 *>(tile_hi + C::A_TILE + off) = l;
        }
      }
    };

    float acc[C::ACC], accx[C::ACC], tot[C::ACC];  // hi x hi of the current tap | cross terms | hi x hi of done taps
#pragma unroll
    for (int i = 0; i < C::ACC; ++i) acc[i] = accx[i] = tot[i] = 0.f;
    for (int q = 0; q < S - 1; ++q) {
      issue(q);
      if constexpr (SPLIT_ROWS) cp_async_commit();
    }
    for (int u = 0; u < n_uses; ++u) {
      const uint32_t slot = (gu + static_cast<uint32_t>(u)) % S, par = ((gu + static_cast<uint32_t>(u)) / S) & 1u;
      if constexpr (SPLIT_ROWS) cp_async_wait<S - 2>();  // this thread's gathers of use u have landed
      fence_proxy_async();  // this thread's generic-proxy writes of the A tiles -> wgmma (async proxy) reads
      mbar_wait(smem_u32(&s_full[slot]), par);
      __syncthreads();      // whole stage present; the wgmma of use u - 1 have retired in both warpgroups
      const uint32_t a_hi = ring + slot * C::STAGE + static_cast<uint32_t>(wg * 64 * (C::KC * 4)), a_lo = a_hi + C::A_TILE;
      const uint32_t b_hi = ring + slot * C::STAGE + C::A_STAGE, b_lo = b_hi + COUT * 16;  // rows 0..N-1 = hi, N..2N-1 = lo
      const uint32_t tap_first = (u % C::G) == 0;  // the tap's hi x hi partial starts over (scale_d = 0)
      wg_fence();
#pragma unroll
      for (int j = 0; j < C::KC / 8; ++j) {
        // k-step j: 32 bytes further into the swizzled rows; B: 16-channel block j / 2, chunk pair (j & 1) inside it
        const uint32_t bo = static_cast<uint32_t>(2 * j) * (2 * COUT * 16);
        const uint64_t dah = C::KC == 32 ? desc_sw128(a_hi + j * 32) : desc_sw64(a_hi + j * 32);
        const uint64_t dal = C::KC == 32 ? desc_sw128(a_lo + j * 32) : desc_sw64(a_lo + j * 32);
        const uint64_t dbh = smem_desc(b_hi + bo, 2 * COUT * 16, 128), dbl = smem_desc(b_lo + bo, 2 * COUT * 16, 128);
        wg::mma_tf32<COUT>(accx, dal, dbh, 1u);  // A_lo x B_hi
        wg::mma_tf32<COUT>(accx, dah, dbl, 1u);  // A_hi x B_lo
        wg::mma_tf32<COUT>(acc, dah, dbh, (tap_first && j == 0) ? 0u : 1u);  // A_hi x B_hi
      }
      wg_commit();
      issue(u + S - 1);  // the slot of use u - 1
      if constexpr (SPLIT_ROWS) cp_async_commit();
      wg_wait<0>();
      if (u % C::G == C::G - 1) {  // last chunk of the tap: its partial joins the total
        wg_fence_acc<C::ACC>(acc);
#pragma unroll
        for (int i = 0; i < C::ACC; ++i) tot[i] += acc[i];
      }
    }
    wg_fence_acc<C::ACC>(accx);
    if constexpr (SPLIT_ROWS) cp_async_wait<0>();
    gu += static_cast<uint32_t>(n_uses);

    // ---------------------------------------------------------------- epilogue (accumulator fragment)
#pragma unroll
    for (int i = 0; i < C::ACC; i += 2) {
      const int r = wg * 64 + frag_row(i, wtid), c = frag_col(i, wtid);
      if (r >= rows) continue;
      const size_t orow = static_cast<size_t>(row0 + r);
      float o[2] = {accx[i] + tot[i], accx[i + 1] + tot[i + 1]};
      float res[2] = {0.f, 0.f};
      if (residual) {
        if constexpr (SPLIT_ROWS) {
          const float2 h = __ldg(reinterpret_cast<const float2 *>(residual + orow * (2 * COUT) + c));
          const float2 l = __ldg(reinterpret_cast<const float2 *>(residual + orow * (2 * COUT) + COUT + c));
          res[0] = h.x + l.x;
          res[1] = h.y + l.y;
        } else {
          const float2 rv = __ldg(reinterpret_cast<const float2 *>(residual + orow * COUT + c));
          res[0] = rv.x;
          res[1] = rv.y;
        }
      }
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float v = o[e];
        if (scale) v = v * __ldg(scale + c + e);
        if (shift) v = v + __ldg(shift + c + e);
        if (residual) v = v + res[e];
        if (relu) v = fmaxf(v, 0.f);
        o[e] = v;
      }
      if (out_rows) *reinterpret_cast<float2 *>(out_rows + orow * COUT + c) = make_float2(o[0], o[1]);
      if (SPLIT_ROWS && out_split) {
        float h[2], l[2];
        split_tf32(o[0], h[0], l[0]);
        split_tf32(o[1], h[1], l[1]);
        *reinterpret_cast<float2 *>(out_split + orow * (2 * COUT) + c) = make_float2(h[0], h[1]);
        *reinterpret_cast<float2 *>(out_split + orow * (2 * COUT) + COUT + c) = make_float2(l[0], l[1]);
      }
    }
  }
}

// split-K finalize: v = act((sum_s partial[s][r][c]) * scale + shift (+ residual)), slabs added in index order; the
// residual comes in the conv's row layout, the result goes out as fp32 rows and / or (SPLIT_ROWS) split rows.
template <bool SPLIT_ROWS>
__global__ void __launch_bounds__(256)
    rows_finalize_kernel(const float *__restrict__ partial, int splits, const int32_t *__restrict__ n_dev,
                         long long n_cap, int C, const float *__restrict__ scale, const float *__restrict__ shift,
                         const float *__restrict__ residual, int relu, float *__restrict__ out_f32,
                         float *__restrict__ out_split) {
  // this grid may start while the split-K conv drains (it waits here for the partial sums), and the next layer's
  // prologue may start while this grid runs
  pdl_trigger();
  pdl_wait();
  const long long n = n_dev ? min(static_cast<long long>(n_dev[0]), n_cap) : n_cap;
  const int c4 = C / 4;
  const size_t slab = static_cast<size_t>(n_cap) * C / 4;
  // persistent grid-stride loop over float4s: the grid is sized for the SMs, the trip count follows the device row count
  for (long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; q < n * c4;
       q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = q / c4;
    const int c = static_cast<int>(q - r * c4) * 4;
    const float4 *p = reinterpret_cast<const float4 *>(partial) + q;
    float4 a = __ldg(p);
    for (int s = 1; s < splits; ++s) {
      const float4 b = __ldg(p + s * slab);
      a.x += b.x;
      a.y += b.y;
      a.z += b.z;
      a.w += b.w;
    }
    float v[4] = {a.x, a.y, a.z, a.w};
    float res[4] = {0.f, 0.f, 0.f, 0.f};
    if (residual) {
      if constexpr (SPLIT_ROWS) {
        const float4 h = __ldg(reinterpret_cast<const float4 *>(residual + r * 2 * C + c));
        const float4 l = __ldg(reinterpret_cast<const float4 *>(residual + r * 2 * C + C + c));
        res[0] = h.x + l.x;
        res[1] = h.y + l.y;
        res[2] = h.z + l.z;
        res[3] = h.w + l.w;
      } else {
        const float4 rv = __ldg(reinterpret_cast<const float4 *>(residual) + q);
        res[0] = rv.x;
        res[1] = rv.y;
        res[2] = rv.z;
        res[3] = rv.w;
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (scale) v[j] = v[j] * __ldg(scale + c + j);
      if (shift) v[j] = v[j] + __ldg(shift + c + j);
      if (residual) v[j] = v[j] + res[j];
      if (relu) v[j] = fmaxf(v[j], 0.f);
    }
    if (out_f32) reinterpret_cast<float4 *>(out_f32)[q] = make_float4(v[0], v[1], v[2], v[3]);
    if (SPLIT_ROWS && out_split) {
      float h[4], l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) split_tf32(v[j], h[j], l[j]);
      *reinterpret_cast<float4 *>(out_split + r * 2 * C + c) = make_float4(h[0], h[1], h[2], h[3]);
      *reinterpret_cast<float4 *>(out_split + r * 2 * C + C + c) = make_float4(l[0], l[1], l[2], l[3]);
    }
  }
}

template <int CIN, int COUT, bool SPLIT_ROWS>
int launch(const float *in, const int32_t *nbr, const int32_t *n_out_dev, int64_t n_cap, int K, const float *packed,
           const float *scale, const float *shift, const float *residual, int relu, float *out_f32, float *out_split,
           int splits, cudaStream_t st) {
  using C = Cfg<CIN, COUT, SPLIT_ROWS>;
  const size_t smem = static_cast<size_t>(C::STAGES) * C::STAGE + static_cast<size_t>(kM) * K * sizeof(int32_t) + 1024;
  if (smem > 227 * 1024) return P3D_ERR_UNSUPPORTED;
  auto kern = gather_gemm_tf32_kernel<CIN, COUT, SPLIT_ROWS>;
  P3D_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  const long long work = ((n_cap + kM - 1) / kM) * splits;
  const long long slots = static_cast<long long>(num_sms()) * C::MIN_CTAS;
  P3D_CUDA_CHECK(launch_pdl(kern, dim3(static_cast<unsigned int>(work < slots ? work : slots)), dim3(kThreads), smem, st,
                            in, nbr, n_out_dev, static_cast<long long>(n_cap), K, splits, packed, scale, shift, residual,
                            relu, out_f32, out_split));
  return P3D_OK;
}

// packed[tap][k-chunk ci / 4][hl * Cout + n][ci % 4] = split(W[tap][ci][n]): per 4 input channels a K-major operand of
// 2*Cout rows (tf32 hi rows, then lo rows), so B_lo is the B_hi descriptor advanced by Cout rows and the slice of any
// KC consecutive channels of a tap is one contiguous block.
__global__ void __launch_bounds__(256) pack_weights_kernel(const float *__restrict__ w, int K, int Cin, int Cout,
                                                           float *__restrict__ packed) {
  const long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(K) * Cin * Cout;
  if (q >= total) return;
  const int n = static_cast<int>(q % Cout);
  const int ci = static_cast<int>((q / Cout) % Cin);
  const int t = static_cast<int>(q / (static_cast<long long>(Cout) * Cin));
  float hi, lo;
  split_tf32(w[q], hi, lo);
  const size_t base = (static_cast<size_t>(t) * Cin + (ci & ~3)) * (2 * Cout) + (ci & 3);
  packed[base + static_cast<size_t>(n) * 4] = hi;
  packed[base + static_cast<size_t>(Cout + n) * 4] = lo;
}

// rows [n, C] fp32 <-> split rows [n][2][C]
__global__ void __launch_bounds__(256) rows_split_kernel(const float *__restrict__ x, const int32_t *__restrict__ n_dev,
                                                         long long n_cap, int C, float *__restrict__ out_split) {
  const long long n = n_dev ? min(static_cast<long long>(n_dev[0]), n_cap) : n_cap;
  const long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (q >= n * C) return;
  const long long r = q / C;
  const int c = static_cast<int>(q - r * C);
  float h, l;
  split_tf32(x[q], h, l);
  out_split[r * 2 * C + c] = h;
  out_split[r * 2 * C + C + c] = l;
}
__global__ void __launch_bounds__(256) rows_merge_kernel(const float *__restrict__ xs, const int32_t *__restrict__ n_dev,
                                                         long long n_cap, int C, float *__restrict__ out) {
  const long long n = n_dev ? min(static_cast<long long>(n_dev[0]), n_cap) : n_cap;
  const long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (q >= n * C) return;
  const long long r = q / C;
  const int c = static_cast<int>(q - r * C);
  out[q] = xs[r * 2 * C + c] + xs[r * 2 * C + C + c];
}

}  // namespace tc
}  // namespace p3d

using namespace p3d;

// Both row layouts after their entry point's argument checks: split-K choice, conv launch, finalize.
static int gather_gemm(bool split_rows, const float *in, const int32_t *nbr, const int32_t *n_out_dev, int64_t n_out_cap,
                       int K, int Cin, int Cout, const float *packed_weight, const float *scale, const float *shift,
                       const float *residual, int relu, float *out_f32, float *out_split, void *workspace,
                       size_t workspace_bytes, cudaStream_t st) {
  int splits = tc::splits_for(Cout);
  if (splits > K) splits = K;
  const size_t need = static_cast<size_t>(splits) * static_cast<size_t>(n_out_cap) * Cout * sizeof(float);
  const bool split = splits > 1 && workspace && workspace_bytes >= need;
  float *k_f32 = split ? static_cast<float *>(workspace) : out_f32, *k_split = split ? nullptr : out_split;
  const float *k_scale = split ? nullptr : scale, *k_shift = split ? nullptr : shift, *k_res = split ? nullptr : residual;
  const int k_relu = split ? 0 : relu, k_splits = split ? splits : 1;
  int rc = P3D_ERR_UNSUPPORTED;
#define P3D_TC_CASE(CI, CO)                                                                                               \
  if (Cin == CI && Cout == CO)                                                                                            \
    rc = split_rows ? tc::launch<CI, CO, true>(in, nbr, n_out_dev, n_out_cap, K, packed_weight, k_scale, k_shift, k_res,  \
                                               k_relu, k_f32, k_split, k_splits, st)                                      \
                    : tc::launch<CI, CO, false>(in, nbr, n_out_dev, n_out_cap, K, packed_weight, k_scale, k_shift, k_res, \
                                                k_relu, k_f32, k_split, k_splits, st);
  P3D_TC_CASE(16, 16)
  P3D_TC_CASE(16, 32)
  P3D_TC_CASE(32, 32)
  P3D_TC_CASE(32, 64)
  P3D_TC_CASE(64, 64)
  P3D_TC_CASE(64, 128)
  P3D_TC_CASE(128, 128)
#undef P3D_TC_CASE
  if (rc != P3D_OK || !split) return rc;
  const long long fin_blocks = (n_out_cap * (Cout / 4) + 255) / 256;
  const float *partial = k_f32;
  P3D_CUDA_CHECK(launch_pdl(split_rows ? tc::rows_finalize_kernel<true> : tc::rows_finalize_kernel<false>,
                            dim3(static_cast<unsigned int>(fin_blocks < num_sms() * 8 ? fin_blocks : num_sms() * 8)),
                            dim3(256), 0, st, partial, splits, n_out_dev, static_cast<long long>(n_out_cap), Cout, scale,
                            shift, residual, relu, out_f32, out_split));
  return P3D_OK;
}

extern "C" size_t p3d_sparse_conv_packed_weight_bytes(int K, int Cin, int Cout) {
  if (K < 1 || Cin < 16 || Cout < 16 || Cin % 16 || Cout % 16) return 0;
  return align_up(static_cast<size_t>(K) * Cin * Cout * 2 * sizeof(float));
}

extern "C" int p3d_sparse_conv_pack_weights(const float *weight, int K, int Cin, int Cout, float *packed,
                                            p3d_stream_t stream) {
  if (!weight || !packed || K < 1) return P3D_ERR_INVALID_ARG;
  if (Cin < 16 || Cout < 16 || Cin % 16 || Cout % 16) return P3D_ERR_UNSUPPORTED;
  const long long total = static_cast<long long>(K) * Cin * Cout;
  tc::pack_weights_kernel<<<div_up(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(weight, K, Cin, Cout,
                                                                                            packed);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" size_t p3d_sparse_conv_splitk_workspace_bytes(int64_t n_out_cap, int Cin, int Cout) {
  (void)Cin;
  if (n_out_cap <= 0 || Cout < 16) return 0;
  const int s = tc::splits_for(Cout);
  return s > 1 ? align_up(static_cast<size_t>(s) * static_cast<size_t>(n_out_cap) * Cout * sizeof(float)) : 0;
}

extern "C" int p3d_sparse_conv_gather_gemm_tf32x3_ws(const float *in, const int32_t *nbr, const int32_t *n_out_dev,
                                                     int64_t n_out_cap, int K, int Cin, int Cout, const float *weight,
                                                     const float *scale, const float *shift, const float *residual,
                                                     int relu, float *out, void *workspace, size_t workspace_bytes,
                                                     p3d_stream_t stream) {
  if (n_out_cap < 0 || K < 1 || K > 32 || !weight || (n_out_cap && (!in || !nbr || !out))) return P3D_ERR_INVALID_ARG;
  if (n_out_cap == 0) return P3D_OK;
  if ((reinterpret_cast<uintptr_t>(in) & 15) || (reinterpret_cast<uintptr_t>(out) & 15) ||
      (reinterpret_cast<uintptr_t>(weight) & 15) || (reinterpret_cast<uintptr_t>(residual) & 15) ||
      (reinterpret_cast<uintptr_t>(workspace) & 15))
    return P3D_ERR_INVALID_ARG;
  return gather_gemm(false, in, nbr, n_out_dev, n_out_cap, K, Cin, Cout, weight, scale, shift, residual, relu, out,
                     nullptr, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

extern "C" int p3d_sparse_conv_gather_gemm_tf32x3(const float *in, const int32_t *nbr, const int32_t *n_out_dev,
                                                  int64_t n_out_cap, int K, int Cin, int Cout, const float *weight,
                                                  const float *scale, const float *shift, const float *residual,
                                                  int relu, float *out, p3d_stream_t stream) {
  return p3d_sparse_conv_gather_gemm_tf32x3_ws(in, nbr, n_out_dev, n_out_cap, K, Cin, Cout, weight, scale, shift, residual,
                                               relu, out, nullptr, 0, stream);
}

extern "C" int p3d_rows_convert_layout(const float *src, int src_layout, const int32_t *n_dev, int64_t n_cap, int C,
                                       float *dst, p3d_stream_t stream) {
  if (n_cap < 0 || C < 1 || (n_cap && (!src || !dst)) || (src_layout != 0 && src_layout != 1)) return P3D_ERR_INVALID_ARG;
  if (n_cap == 0) return P3D_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (src_layout == 0)
    tc::rows_split_kernel<<<div_up(n_cap * C, 256), 256, 0, st>>>(src, n_dev, n_cap, C, dst);
  else
    tc::rows_merge_kernel<<<div_up(n_cap * C, 256), 256, 0, st>>>(src, n_dev, n_cap, C, dst);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" int p3d_sparse_conv_gather_gemm_split_ws(const float *in_split, const int32_t *nbr,
                                                    const int32_t *n_out_dev, int64_t n_out_cap, int K, int Cin,
                                                    int Cout, const float *packed_weight, const float *scale,
                                                    const float *shift, const float *residual_split, int relu,
                                                    float *out_f32, float *out_split, void *workspace,
                                                    size_t workspace_bytes, p3d_stream_t stream) {
  if (n_out_cap < 0 || K < 1 || K > 32 || !packed_weight || (!out_f32 && !out_split) || (n_out_cap && (!in_split || !nbr)))
    return P3D_ERR_INVALID_ARG;
  if (n_out_cap == 0) return P3D_OK;
  if ((reinterpret_cast<uintptr_t>(in_split) & 15) || (reinterpret_cast<uintptr_t>(out_f32) & 15) ||
      (reinterpret_cast<uintptr_t>(out_split) & 15) || (reinterpret_cast<uintptr_t>(packed_weight) & 15) ||
      (reinterpret_cast<uintptr_t>(residual_split) & 15) || (reinterpret_cast<uintptr_t>(workspace) & 15) ||
      (reinterpret_cast<uintptr_t>(nbr) & 15))
    return P3D_ERR_INVALID_ARG;
  return gather_gemm(true, in_split, nbr, n_out_dev, n_out_cap, K, Cin, Cout, packed_weight, scale, shift, residual_split,
                     relu, out_f32, out_split, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

extern "C" int p3d_sparse_conv_gather_gemm_split(const float *in_split, const int32_t *nbr, const int32_t *n_out_dev,
                                                 int64_t n_out_cap, int K, int Cin, int Cout, const float *packed_weight,
                                                 const float *scale, const float *shift, const float *residual_split,
                                                 int relu, float *out_f32, float *out_split, p3d_stream_t stream) {
  return p3d_sparse_conv_gather_gemm_split_ws(in_split, nbr, n_out_dev, n_out_cap, K, Cin, Cout, packed_weight, scale,
                                              shift, residual_split, relu, out_f32, out_split, nullptr, 0, stream);
}
