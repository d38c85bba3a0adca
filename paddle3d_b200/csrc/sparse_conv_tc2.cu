// Sparse-conv gather-GEMM on wgmma, split-row version: activations travel between layers already split into their
// tf32 hi / lo halves (row layout [n][2][C]: hi row, then lo row), so the 3xTF32 split is paid ONCE per produced
// element (in the producing layer's epilogue) instead of once per gathering neighbour (11-27x), and the gather
// becomes a pure copy that cp.async (LDGSTS, 16 B, zero-fill for missing neighbours) drops straight into swizzled
// wgmma operand tiles — no register staging, no ALU on the data in the gather.
//
//   grid        persistent: min(#work items at capacity, MIN_CTAS x SMs) CTAs, each walks the work items
//               w = blockIdx.x, +gridDim.x, ... (w = tile * splits + split) of the DEVICE row count.
//   CTA         two warpgroups; warpgroup g owns rows 64g .. 64g+63 of the 128-row tile (one m64nCout accumulator).
//   gather      per (tap, KC-channel chunk) "use", full-128-byte-line cp.async gathers (8 threads per line, 32 rows
//               per CTA instruction) into SWIZZLE_128B (KC = 32) or SWIZZLE_64B (KC = 16) tiles, STAGES - 1 uses ahead;
//               thread 0 copies the packed [hi | lo] weight slice of the use with cp.async.bulk (mbarrier complete_tx).
//               TMA = true (Cin >= 32): warp 0 gathers the rows with one 2-D TMA box (one 128-byte line) per row half
//               instead; a missing neighbour (row -1) is out of bounds for the tensor map and arrives as zeros.
//   mma         3 wgmma kind tf32 per 8-wide k-step: hi x hi into one accumulator, lo x hi + hi x lo into a second one.
//   epilogue    BN scale/shift (+bias), residual (= hi + lo of the split residual rows), ReLU, then plain fp32 rows,
//               split rows for the next layer, or both, from the accumulator fragment.
#include <cuda.h>  // CUtensorMap (types only: the encoder is fetched with cudaGetDriverEntryPoint)

#include "tc_common.cuh"

namespace p3d {
namespace tc2 {

using namespace tc;

template <int CIN, int COUT>
struct Cfg {
  // One pipeline "use" = one tap x KC input channels for the CTA's 128 rows.
  static constexpr int KC = (CIN >= 32) ? 32 : 16;        // 32 channels = one full 128-byte line per gathered row half
  static constexpr int G = CIN / KC;
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

// 2-D TMA box of the split rows' tensor map (one 128-byte line of one row) into a SWIZZLE_128B tile row
__device__ __forceinline__ void tma_row(uint32_t dst, const CUtensorMap *map, int col, int row, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(col), "r"(row), "r"(bar)
      : "memory");
}

__device__ __forceinline__ int nth_bit(uint32_t m, int k) {  // position of the k-th (0-based) set bit of m
  for (int i = 0; i < k; ++i) m &= m - 1u;
  return __ffs(m) - 1;
}

template <int CIN, int COUT, bool TMA>
__global__ void __launch_bounds__(kThreads, Cfg<CIN, COUT>::MIN_CTAS)
    gather_gemm_split_kernel(const __grid_constant__ CUtensorMap in_map, const float *__restrict__ in_split,
                             const int32_t *__restrict__ nbr,
                             const int32_t *__restrict__ n_out_dev, long long n_cap, int K, int splits,
                             const float *__restrict__ packed_w, const float *__restrict__ scale,
                             const float *__restrict__ shift, const float *__restrict__ residual_split, int relu,
                             float *__restrict__ out_f32, float *__restrict__ out_split) {
  using C = Cfg<CIN, COUT>;
  constexpr int S = C::STAGES;
  // Programmatic dependent launch: let the next kernel of the stream start its prologue while this grid drains.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");  // inputs of the previous layer are complete
  const long long n = n_out_dev ? min(static_cast<long long>(n_out_dev[0]), n_cap) : n_cap;
  // work items w = tile * splits + split; split s owns the taps t == s (mod splits) and, when splits > 1, writes raw
  // partial sums to slab s of out_f32 (the caller passes the scratch slabs and no epilogue operands).
  const long long n_work = ((n + kM - 1) / kM) * splits;
  if (static_cast<long long>(blockIdx.x) >= n_work) return;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  int32_t *s_nbr = reinterpret_cast<int32_t *>(smem + C::STAGES * C::STAGE);  // [kM][K]
  __shared__ __align__(8) unsigned long long s_bar[8 + 1];  // full[8] (weights, and the rows with TMA) nbr_loaded
  constexpr int kF = 0, kNB = 8;
  __shared__ uint32_t s_active;

  const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7, wtid = tid & 127;
  if (tid == 0) {
    for (int s = 0; s < S; ++s) mbar_init(smem_u32(&s_bar[kF + s]), 1);
    mbar_init(smem_u32(&s_bar[kNB]), 1);
    fence_mbar_init();
  }
  __syncthreads();
  const uint32_t ring = smem_u32(smem);

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
      const uint32_t words = static_cast<uint32_t>(avail) * K, bulk_words = words & ~3u;
      if (tid == 0) {
        fence_proxy_async();  // earlier generic reads of s_nbr vs the async-proxy write
        mbar_arrive_expect_tx(smem_u32(&s_bar[kNB]), bulk_words * 4);
        if (bulk_words) bulk_g2s(smem_u32(s_nbr), nbr + row0 * K, bulk_words * 4, smem_u32(&s_bar[kNB]));
      }
      if (bulk_words + tid < words) s_nbr[bulk_words + tid] = __ldg(nbr + row0 * K + bulk_words + tid);
      __syncthreads();  // s_active reset and the up-to-3 tail words are plain stores
      mbar_wait(smem_u32(&s_bar[kNB]), static_cast<uint32_t>(item_it & 1));
      uint32_t mine = 0u;
      for (int q = tid; q < rows * K; q += kThreads)
        if (s_nbr[q] >= 0) mine |= 1u << (q % K);
      mine = __reduce_or_sync(0xffffffffu, mine);
      if (lane == 0 && mine) atomicOr(&s_active, mine);
    }
    __syncthreads();
    const uint32_t active = s_active & tap_mask;
    const int n_uses = __popc(active) * C::G;

    // gather use q (tap, chunk) of this item into its ring slot; thread 0 posts the weight slice (and the row bytes
    // of the TMA gather) on the slot's barrier
    auto issue = [&](int q) {
      if (q >= n_uses) return;
      const int t = nth_bit(active, q / C::G), g = q % C::G;
      const uint32_t slot = (gu + static_cast<uint32_t>(q)) % S;
      const uint32_t st = ring + slot * C::STAGE, bar = smem_u32(&s_bar[kF + slot]);
      if (tid == 0) {
        mbar_arrive_expect_tx(bar, static_cast<uint32_t>((TMA ? C::A_STAGE : 0) + C::B_STAGE));
        bulk_g2s(st + C::A_STAGE, packed_w + (static_cast<size_t>(t) * CIN + g * C::KC) * (2 * COUT),
                 static_cast<uint32_t>(C::B_STAGE), bar);
      }
      if (TMA) {
        if (tid < 32) {
          __syncwarp();  // expect_tx is posted before any row can complete
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int row = lane * 4 + k;
            const int src = row < rows ? s_nbr[row * K + t] : -1;
            tma_row(st + row * 128, &in_map, g * 32, src, bar);                   // hi
            tma_row(st + C::A_TILE + row * 128, &in_map, CIN + g * 32, src, bar);  // lo
          }
        }
        return;
      }
      const int sub = tid >> 3;  // 32 rows per CTA instruction
      if (C::KC == 32) {
        // SWIZZLE_128B tiles (row pitch 128 B, chunk ^= row & 7); the hi and the lo line of a row
        const int ch = tid & 7;
#pragma unroll
        for (int q4 = 0; q4 < 4; ++q4) {
          const int row = q4 * 32 + sub;
          const int src = row < rows ? s_nbr[row * K + t] : -1;
          const bool ok = src >= 0;
          const float *p = in_split + (ok ? static_cast<size_t>(src) * (2 * CIN) : 0) + g * 32 + ch * 4;
          const uint32_t d = st + static_cast<uint32_t>(row * 128 + ((ch ^ (row & 7)) << 4));
          cp_async16(d, p, ok);                    // hi
          cp_async16(d + C::A_TILE, p + CIN, ok);  // lo
        }
      } else {
        // 16-channel layers: a split row [hi 16 | lo 16] is ONE line (threads 0-3 of a row fetch the hi chunks,
        // 4-7 the lo chunks); SWIZZLE_64B tiles (row pitch 64 B, chunk ^= (row >> 1) & 3)
        const int ch = tid & 3, part = (tid >> 2) & 1;
#pragma unroll
        for (int q4 = 0; q4 < 4; ++q4) {
          const int row = q4 * 32 + sub;
          const int src = row < rows ? s_nbr[row * K + t] : -1;
          const bool ok = src >= 0;
          const float *p = in_split + (ok ? static_cast<size_t>(src) * (2 * CIN) : 0) + part * CIN + g * 16 + ch * 4;
          const uint32_t d = st + static_cast<uint32_t>(part * C::A_TILE + row * 64 + ((ch ^ ((row >> 1) & 3)) << 4));
          cp_async16(d, p, ok);
        }
      }
    };

    float acc[C::ACC], accx[C::ACC];  // hi x hi | cross terms
#pragma unroll
    for (int i = 0; i < C::ACC; ++i) acc[i] = accx[i] = 0.f;
    for (int q = 0; q < S - 1; ++q) {
      issue(q);
      cp_async_commit();
    }
    for (int u = 0; u < n_uses; ++u) {
      const uint32_t slot = (gu + static_cast<uint32_t>(u)) % S, par = ((gu + static_cast<uint32_t>(u)) / S) & 1u;
      cp_async_wait<S - 2>();  // this thread's gathers of use u have landed
      fence_proxy_async();     // cp.async (generic proxy) writes -> wgmma (async proxy) reads
      mbar_wait(smem_u32(&s_bar[kF + slot]), par);
      __syncthreads();         // whole stage present; the wgmma of use u - 1 have retired in both warpgroups
      const uint32_t a_hi = ring + slot * C::STAGE, a_lo = a_hi + C::A_TILE;
      const uint32_t b_hi = a_hi + C::A_STAGE, b_lo = b_hi + COUT * 16;  // rows 0..N-1 = hi, N..2N-1 = lo
      const uint32_t a_wg = static_cast<uint32_t>(wg * 64 * (C::KC * 4));  // this warpgroup's 64 rows
      wg_fence();
#pragma unroll
      for (int j = 0; j < C::KC / 8; ++j) {
        // k-step j: 32 bytes further into the swizzled rows; B: 16-channel block j / 2, chunk pair (j & 1) inside it
        const uint32_t bo = static_cast<uint32_t>(2 * j) * (2 * COUT * 16);
        uint64_t dah, dal;
        if (C::KC == 32) {
          dah = desc_sw128(a_hi + a_wg + j * 32);
          dal = desc_sw128(a_lo + a_wg + j * 32);
        } else {
          dah = desc_sw64(a_hi + a_wg + j * 32);
          dal = desc_sw64(a_lo + a_wg + j * 32);
        }
        const uint64_t dbh = smem_desc(b_hi + bo, 2 * COUT * 16, 128), dbl = smem_desc(b_lo + bo, 2 * COUT * 16, 128);
        wg::mma_tf32<COUT>(accx, dal, dbh, 1u);  // A_lo x B_hi
        wg::mma_tf32<COUT>(accx, dah, dbl, 1u);  // A_hi x B_lo
        wg::mma_tf32<COUT>(acc, dah, dbh, 1u);  // A_hi x B_hi
      }
      wg_commit();
      issue(u + S - 1);  // the slot of use u - 1
      cp_async_commit();
      wg_wait<0>();
    }
    wg_fence_acc<C::ACC>(acc);
    wg_fence_acc<C::ACC>(accx);
    cp_async_wait<0>();
    gu += static_cast<uint32_t>(n_uses);

    // ---------------------------------------------------------------- epilogue (accumulator fragment)
#pragma unroll
    for (int i = 0; i < C::ACC; i += 2) {
      const int r = wg * 64 + frag_row(i, wtid), c = frag_col(i, wtid);
      if (r >= rows) continue;
      const size_t orow = static_cast<size_t>(row0 + r);
      float o[2] = {accx[i] + acc[i], accx[i + 1] + acc[i + 1]};
      float res[2] = {0.f, 0.f};
      if (residual_split) {
        const float2 h = __ldg(reinterpret_cast<const float2 *>(residual_split + orow * (2 * COUT) + c));
        const float2 l = __ldg(reinterpret_cast<const float2 *>(residual_split + orow * (2 * COUT) + COUT + c));
        res[0] = h.x + l.x;
        res[1] = h.y + l.y;
      }
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float v = o[e];
        if (scale) v = v * __ldg(scale + c + e);
        if (shift) v = v + __ldg(shift + c + e);
        if (residual_split) v = v + res[e];
        if (relu) v = fmaxf(v, 0.f);
        o[e] = v;
      }
      if (out_rows) *reinterpret_cast<float2 *>(out_rows + orow * COUT + c) = make_float2(o[0], o[1]);
      if (out_split) {
        float h[2], l[2];
        split_tf32(o[0], h[0], l[0]);
        split_tf32(o[1], h[1], l[1]);
        *reinterpret_cast<float2 *>(out_split + orow * (2 * COUT) + c) = make_float2(h[0], h[1]);
        *reinterpret_cast<float2 *>(out_split + orow * (2 * COUT) + COUT + c) = make_float2(l[0], l[1]);
      }
    }
  }
}

// Tensor map of the split rows [n_rows][2 * C] fp32 for tile::gather4: box = 32 columns (one 128-byte line) x 1 row,
// SWIZZLE_128B, out-of-bounds reads (missing neighbours) filled with zeros.
inline int make_rows_map(const float *rows, int64_t n_rows, int C, CUtensorMap *map) {
  using Encode = CUresult (*)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                              const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static Encode encode = nullptr;
  if (!encode) {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) != cudaSuccess || !fn)
      return P3D_ERR_UNSUPPORTED;
    encode = reinterpret_cast<Encode>(fn);
  }
  const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(2 * C), static_cast<cuuint64_t>(n_rows)};
  const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(2 * C) * sizeof(float)};
  const cuuint32_t box[2] = {32u, 1u}, estride[2] = {1u, 1u};
  const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float *>(rows), gdim, gstride, box, estride,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? P3D_OK : P3D_ERR_INVALID_ARG;
}

template <int CIN, int COUT, bool TMA = false>
int launch(const float *in_split, const int32_t *nbr, const int32_t *n_out_dev, int64_t n_cap, int K,
           const float *packed, const float *scale, const float *shift, const float *residual_split, int relu,
           float *out_f32, float *out_split, cudaStream_t st, int splits = 1, int64_t n_in_rows = 0) {
  using C = Cfg<CIN, COUT>;
  CUtensorMap in_map = {};
  if (TMA) {
    static_assert(!TMA || C::KC == 32, "the TMA gather is written for 32-channel uses");
    const int rc = make_rows_map(in_split, n_in_rows, CIN, &in_map);
    if (rc != P3D_OK) return rc;
  }
  const size_t smem = static_cast<size_t>(C::STAGES) * C::STAGE + static_cast<size_t>(kM) * K * sizeof(int32_t) + 1024;
  if (smem > 227 * 1024) return P3D_ERR_UNSUPPORTED;
  auto kern = gather_gemm_split_kernel<CIN, COUT, TMA>;
  P3D_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  const long long work = ((n_cap + kM - 1) / kM) * splits;
  const long long slots = static_cast<long long>(num_sms()) * C::MIN_CTAS;
  const unsigned int grid = static_cast<unsigned int>(work < slots ? work : slots);
  static const bool pdl = !(getenv("P3D_PDL") && atoi(getenv("P3D_PDL")) == 0);  // tuning hook, default on
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  const long long n_cap_ll = n_cap;
  P3D_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, in_map, in_split, nbr, n_out_dev, n_cap_ll, K, splits, packed, scale, shift,
                                    residual_split, relu, out_f32, out_split));
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

// split-K finalize: v = act((sum_s partial[s][r][c]) * scale + shift (+ residual)), slabs added in index order; the
// residual comes in the split layout and the result goes out as fp32 rows and / or split rows.
__global__ void __launch_bounds__(256)
    rows_finalize_split_kernel(const float *__restrict__ partial, int splits, const int32_t *__restrict__ n_dev,
                               long long n_cap, int C, const float *__restrict__ scale, const float *__restrict__ shift,
                               const float *__restrict__ residual_split, int relu, float *__restrict__ out_f32,
                               float *__restrict__ out_split) {
  // programmatic dependent launch on both sides: this grid may start while the split-K conv drains (it waits here
  // for the partial sums), and the next layer's prologue may start while this grid runs
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const long long n = n_dev ? min(static_cast<long long>(n_dev[0]), n_cap) : n_cap;
  const int c4 = C / 4;
  const size_t slab = static_cast<size_t>(n_cap) * C / 4;
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
    if (residual_split) {
      const float4 h = __ldg(reinterpret_cast<const float4 *>(residual_split + r * 2 * C + c));
      const float4 l = __ldg(reinterpret_cast<const float4 *>(residual_split + r * 2 * C + C + c));
      res[0] = h.x + l.x;
      res[1] = h.y + l.y;
      res[2] = h.z + l.z;
      res[3] = h.w + l.w;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (scale) v[j] = v[j] * __ldg(scale + c + j);
      if (shift) v[j] = v[j] + __ldg(shift + c + j);
      if (residual_split) v[j] = v[j] + res[j];
      if (relu) v[j] = fmaxf(v[j], 0.f);
    }
    if (out_f32) reinterpret_cast<float4 *>(out_f32)[q] = make_float4(v[0], v[1], v[2], v[3]);
    if (out_split) {
      float h[4], l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) split_tf32(v[j], h[j], l[j]);
      *reinterpret_cast<float4 *>(out_split + r * 2 * C + c) = make_float4(h[0], h[1], h[2], h[3]);
      *reinterpret_cast<float4 *>(out_split + r * 2 * C + C + c) = make_float4(l[0], l[1], l[2], l[3]);
    }
  }
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

}  // namespace tc2
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_rows_convert_layout(const float *src, int src_layout, const int32_t *n_dev, int64_t n_cap, int C,
                                       float *dst, p3d_stream_t stream) {
  if (n_cap < 0 || C < 1 || (n_cap && (!src || !dst)) || (src_layout != 0 && src_layout != 1)) return P3D_ERR_INVALID_ARG;
  if (n_cap == 0) return P3D_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (src_layout == 0)
    tc2::rows_split_kernel<<<div_up(n_cap * C, 256), 256, 0, st>>>(src, n_dev, n_cap, C, dst);
  else
    tc2::rows_merge_kernel<<<div_up(n_cap * C, 256), 256, 0, st>>>(src, n_dev, n_cap, C, dst);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

static int split_conv(const float *in_split, int64_t n_in_rows, bool tma, const int32_t *nbr, const int32_t *n_out_dev,
                      int64_t n_out_cap, int K, int Cin, int Cout, const float *packed_weight, const float *scale,
                      const float *shift, const float *residual_split, int relu, float *out_f32, float *out_split,
                      void *workspace, size_t workspace_bytes, p3d_stream_t stream) {
  if (n_out_cap < 0 || K < 1 || K > 32 || !packed_weight || (!out_f32 && !out_split) || (n_out_cap && (!in_split || !nbr)))
    return P3D_ERR_INVALID_ARG;
  if (n_out_cap == 0) return P3D_OK;
  if ((reinterpret_cast<uintptr_t>(in_split) & 15) || (reinterpret_cast<uintptr_t>(out_f32) & 15) ||
      (reinterpret_cast<uintptr_t>(out_split) & 15) || (reinterpret_cast<uintptr_t>(packed_weight) & 15) ||
      (reinterpret_cast<uintptr_t>(residual_split) & 15) || (reinterpret_cast<uintptr_t>(workspace) & 15) ||
      (reinterpret_cast<uintptr_t>(nbr) & 15))
    return P3D_ERR_INVALID_ARG;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // split-K over taps for the layers with few 128-row tiles (same policy and scratch size as the fp32-row kernel)
  int splits = tc::splits_for(Cout);
  if (splits > K) splits = K;
  const size_t need = static_cast<size_t>(splits) * static_cast<size_t>(n_out_cap) * Cout * sizeof(float);
  const bool split = splits > 1 && workspace && workspace_bytes >= need;
  float *k_f32 = split ? static_cast<float *>(workspace) : out_f32, *k_split = split ? nullptr : out_split;
  const float *k_scale = split ? nullptr : scale, *k_shift = split ? nullptr : shift;
  const float *k_res = split ? nullptr : residual_split;
  const int k_relu = split ? 0 : relu, k_splits = split ? splits : 1;
  int rc = P3D_ERR_UNSUPPORTED;
#define P3D_TC2_CASE(CI, CO)                                                                                           \
  if (!tma && Cin == CI && Cout == CO)                                                                                 \
    rc = tc2::launch<CI, CO>(in_split, nbr, n_out_dev, n_out_cap, K, packed_weight, k_scale, k_shift, k_res, k_relu,    \
                             k_f32, k_split, st, k_splits);
#define P3D_TC2_TMA_CASE(CI, CO)                                                                                       \
  if (tma && Cin == CI && Cout == CO)                                                                                  \
    rc = tc2::launch<CI, CO, true>(in_split, nbr, n_out_dev, n_out_cap, K, packed_weight, k_scale, k_shift, k_res,      \
                                   k_relu, k_f32, k_split, st, k_splits, n_in_rows);
  P3D_TC2_CASE(16, 16)
  P3D_TC2_CASE(16, 32)
  P3D_TC2_CASE(32, 32)
  P3D_TC2_CASE(32, 64)
  P3D_TC2_CASE(64, 64)
  P3D_TC2_CASE(64, 128)
  P3D_TC2_CASE(128, 128)
  P3D_TC2_TMA_CASE(32, 32)
  P3D_TC2_TMA_CASE(32, 64)
  P3D_TC2_TMA_CASE(64, 64)
  P3D_TC2_TMA_CASE(64, 128)
  P3D_TC2_TMA_CASE(128, 128)
#undef P3D_TC2_CASE
#undef P3D_TC2_TMA_CASE
  if (rc != P3D_OK || !split) return rc;
  const long long fin_blocks = (n_out_cap * (Cout / 4) + 255) / 256;
  {
    static const bool pdl = !(getenv("P3D_PDL") && atoi(getenv("P3D_PDL")) == 0);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned int>(fin_blocks < num_sms() * 8 ? fin_blocks : num_sms() * 8));
    cfg.blockDim = dim3(256);
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    const float *partial = k_f32;
    const long long cap_ll = n_out_cap;
    P3D_CUDA_CHECK(cudaLaunchKernelEx(&cfg, tc2::rows_finalize_split_kernel, partial, splits, n_out_dev, cap_ll, Cout,
                                      scale, shift, residual_split, relu, out_f32, out_split));
  }
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" int p3d_sparse_conv_gather_gemm_split_ws(const float *in_split, const int32_t *nbr,
                                                    const int32_t *n_out_dev, int64_t n_out_cap, int K, int Cin,
                                                    int Cout, const float *packed_weight, const float *scale,
                                                    const float *shift, const float *residual_split, int relu,
                                                    float *out_f32, float *out_split, void *workspace,
                                                    size_t workspace_bytes, p3d_stream_t stream) {
  return split_conv(in_split, 0, false, nbr, n_out_dev, n_out_cap, K, Cin, Cout, packed_weight, scale, shift,
                    residual_split, relu, out_f32, out_split, workspace, workspace_bytes, stream);
}

extern "C" int p3d_sparse_conv_gather_gemm_split_tma(const float *in_split, int64_t n_in_rows, const int32_t *nbr,
                                                     const int32_t *n_out_dev, int64_t n_out_cap, int K, int Cin,
                                                     int Cout, const float *packed_weight, const float *scale,
                                                     const float *shift, const float *residual_split, int relu,
                                                     float *out_f32, float *out_split, void *workspace,
                                                     size_t workspace_bytes, p3d_stream_t stream) {
  if (n_in_rows < 1 || Cin < 32) return P3D_ERR_UNSUPPORTED;
  return split_conv(in_split, n_in_rows, true, nbr, n_out_dev, n_out_cap, K, Cin, Cout, packed_weight, scale, shift,
                    residual_split, relu, out_f32, out_split, workspace, workspace_bytes, stream);
}

extern "C" int p3d_sparse_conv_gather_gemm_split(const float *in_split, const int32_t *nbr, const int32_t *n_out_dev,
                                                 int64_t n_out_cap, int K, int Cin, int Cout, const float *packed_weight,
                                                 const float *scale, const float *shift, const float *residual_split,
                                                 int relu, float *out_f32, float *out_split, p3d_stream_t stream) {
  return p3d_sparse_conv_gather_gemm_split_ws(in_split, nbr, n_out_dev, n_out_cap, K, Cin, Cout, packed_weight, scale,
                                              shift, residual_split, relu, out_f32, out_split, nullptr, 0, stream);
}
