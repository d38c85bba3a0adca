// Sparse-conv gather-GEMM on Hopper tensor cores: wgmma kind tf32, fp32 accumulators in registers,
// 3xTF32 split (a = hi + lo, b = hi + lo; D += a_hi*b_hi + a_hi*b_lo + a_lo*b_hi) for fp32-level accuracy.
//
// One CTA (two warpgroups) owns 128 consecutive output rows — warpgroup g the rows 64g .. 64g+63, one m64nCout
// accumulator — and walks the K dimension = (active taps) x (Cin in chunks of KC = 16 channels) through a ring of
// shared-memory stages, STAGES - 1 uses ahead of the tensor cores:
//
//   gather     thread r of the 128 rows (two threads per row, two 16-byte chunks each) loads row nbr[row0 + r][tap]
//              of the input, splits every value into tf32 hi / lo and stores both into the stage's A tiles in the
//              canonical no-swizzle K-major core-matrix layout (8 rows x 16 B per core matrix) — a missing neighbour is a
//              zero row.  Thread 0 fires ONE cp.async.bulk per stage that drops the pre-packed weight slice [hi | lo] for
//              (tap, chunk) into the B tiles (TMA engine, mbarrier complete_tx).  Generic-proxy stores are made visible
//              to the tensor cores with fence.proxy.async before the CTA barrier that precedes the wgmma.
//   mma        per 8-wide k-step 3 wgmma: hi x hi into one accumulator, lo x hi + hi x lo into a second one (the small
//              cross terms keep their own rounding; the epilogue adds the two); the gather of use u + S - 1
//              runs while the wgmma of use u execute, a stage is refilled once the wgmma that read it have retired.
//   epilogue   from the accumulator fragment: fused BN scale/shift (+bias), residual, ReLU, 8-byte row stores.
//
// Taps that no row of the tile uses are skipped for the whole tile (block-uniform bitmask).
// Weights are packed once per layer by p3d_sparse_conv_pack_weights into exactly the shared-memory image:
//   packed[tap][chunk g][hi|lo][KC/4 k-chunks][Cout rows][4 floats].
#include "tc_common.cuh"

namespace p3d {
namespace tc {

template <int CIN, int COUT>
struct Cfg {
  static constexpr int KC = kc_of(CIN);          // channels per stage
  static constexpr int G = CIN / KC;             // stages per tap
  static constexpr int CH = KC / 4;              // 16-byte k-chunks per stage
  static constexpr int A_TILE = KC * kM * 4;     // bytes, one of hi / lo
  static constexpr int B_TILE = KC * COUT * 4;   // bytes, one of hi / lo
  static constexpr int A_STAGE = 2 * A_TILE;     // hi + lo
  static constexpr int B_STAGE = 2 * B_TILE;     // hi + lo (one cp.async.bulk)
  static constexpr int STAGE = A_STAGE + B_STAGE;
  static constexpr int MIN_CTAS = (COUT <= 64) ? 2 : 1;
  static constexpr int BUDGET = (COUT <= 64) ? 96 * 1024 : 192 * 1024;
  static constexpr int S_RAW = BUDGET / STAGE;
  static constexpr int STAGES = S_RAW > 8 ? 8 : (S_RAW < 3 ? 3 : S_RAW);
  static constexpr int ACC = COUT / 2;           // registers of one m64 x COUT accumulator per thread
  static_assert(CIN % 16 == 0 && COUT % 16 == 0 && COUT <= 128, "tensor-core path needs 16-channel multiples");
  static_assert(CH * kM * 4 == 2 * kThreads * 4, "two 16-byte chunks per thread and use");
};

__device__ __forceinline__ int nth_bit(uint32_t m, int k) {  // position of the k-th (0-based) set bit of m
  for (int i = 0; i < k; ++i) m &= m - 1u;
  return __ffs(m) - 1;
}

template <int CIN, int COUT>
__global__ void __launch_bounds__(kThreads, Cfg<CIN, COUT>::MIN_CTAS)
    gather_gemm_tf32x3_kernel(const float *__restrict__ in, const int32_t *__restrict__ nbr,
                              const int32_t *__restrict__ n_out_dev, long long n_cap, int K, int splits,
                              const float *__restrict__ packed_w, const float *__restrict__ scale,
                              const float *__restrict__ shift, const float *__restrict__ residual, int relu,
                              float *__restrict__ out_base) {
  using C = Cfg<CIN, COUT>;
  constexpr int S = C::STAGES;
  // Persistent CTAs: the grid is sized for the SMs (not for the row CAPACITY, which would launch thousands of empty
  // CTAs) and every CTA walks the work items  w = blockIdx.x, +gridDim.x, ...  with  w = tile * splits + split.
  // split-K over taps: split s owns the taps t == s (mod splits) and writes raw partial sums to slab s of `out_base`
  // (the host passes no epilogue parameters then; rows_finalize_kernel adds the slabs in a fixed order).
  const long long n = n_out_dev ? min(static_cast<long long>(n_out_dev[0]), n_cap) : n_cap;
  const long long n_work = ((n + kM - 1) / kM) * splits;
  if (static_cast<long long>(blockIdx.x) >= n_work) return;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  int32_t *s_nbr = reinterpret_cast<int32_t *>(smem + S * C::STAGE);      // [kM][K]
  __shared__ __align__(8) unsigned long long s_full[8];                  // weights of a stage landed
  __shared__ uint32_t s_active;                                          // bit t: some row uses tap t (K <= 32)

  const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7, wtid = tid & 127;
  if (tid == 0) {
    for (int s = 0; s < S; ++s) mbar_init(smem_u32(&s_full[s]), 1);
    fence_mbar_init();
  }
  __syncthreads();
  const uint32_t ring = smem_u32(smem);
  const int g_row = tid & (kM - 1), g_c0 = (tid >> 7) * 2;  // gather: row of the tile, first of two 16-byte chunks

  uint32_t gu = 0;  // uses consumed by earlier work items of this CTA: the ring phases keep running
  for (long long w = blockIdx.x; w < n_work; w += gridDim.x) {
    const long long tile = w / splits;
    const int split = static_cast<int>(w - tile * splits);
    const long long row0 = tile * kM;
    const int rows = static_cast<int>(min(static_cast<long long>(kM), n - row0));
    float *out = out_base + static_cast<size_t>(split) * static_cast<size_t>(n_cap) * COUT;
    __syncthreads();  // previous item drained: s_nbr and s_active free
    if (tid == 0) s_active = 0u;
    __syncthreads();
    {
      uint32_t mine = 0u;
      for (int q = tid; q < kM * K; q += kThreads) {
        const int v = (q < rows * K) ? __ldg(nbr + row0 * K + q) : -1;
        s_nbr[q] = v;
        if (v >= 0) mine |= 1u << (q % K);
      }
      mine = __reduce_or_sync(0xffffffffu, mine);
      if (lane == 0 && mine) atomicOr(&s_active, mine);
    }
    __syncthreads();
    uint32_t tap_mask = 0xffffffffu;
    if (splits > 1) {
      tap_mask = 0u;
      for (int t = split; t < K; t += splits) tap_mask |= 1u << t;
    }
    const uint32_t active = s_active & tap_mask;
    const int n_uses = __popc(active) * C::G;

    // gather use q (tap, chunk) of this item into its ring slot; thread 0 also posts the weight slice
    auto issue = [&](int q) {
      if (q >= n_uses) return;
      const int t = nth_bit(active, q / C::G), g = q % C::G;
      const uint32_t slot = (gu + static_cast<uint32_t>(q)) % S;
      uint8_t *st = smem + slot * C::STAGE;
      if (tid == 0) {
        const uint32_t bar = smem_u32(&s_full[slot]);
        mbar_arrive_expect_tx(bar, static_cast<uint32_t>(C::B_STAGE));
        bulk_g2s(ring + slot * C::STAGE + C::A_STAGE, packed_w + (static_cast<size_t>(t) * C::G + g) * (2 * C::KC * COUT),
                 static_cast<uint32_t>(C::B_STAGE), bar);
      }
      const int src = s_nbr[g_row * K + t];
      float4 v[2];
#pragma unroll
      for (int c = 0; c < 2; ++c)
        v[c] = src >= 0 ? __ldg(reinterpret_cast<const float4 *>(in + static_cast<size_t>(src) * CIN + g * C::KC) + g_c0 + c)
                        : make_float4(0.f, 0.f, 0.f, 0.f);
      // A-tile layout: k-chunk c at c*2048 (LBO), 8-row groups 128 B apart (SBO): the 32 lanes of one store
      // instruction (32 consecutive rows, same chunk) cover 512 contiguous bytes — no bank conflicts.
      const uint32_t a_off = static_cast<uint32_t>((g_row >> 3) * 128 + (g_row & 7) * 16);
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        float4 h, l;
        split_tf32(v[c].x, h.x, l.x);
        split_tf32(v[c].y, h.y, l.y);
        split_tf32(v[c].z, h.z, l.z);
        split_tf32(v[c].w, h.w, l.w);
        *reinterpret_cast<float4 *>(st + (g_c0 + c) * (kM * 16) + a_off) = h;
        *reinterpret_cast<float4 *>(st + C::A_TILE + (g_c0 + c) * (kM * 16) + a_off) = l;
      }
    };

    float acc[C::ACC], accx[C::ACC];  // hi x hi | cross terms
#pragma unroll
    for (int i = 0; i < C::ACC; ++i) acc[i] = accx[i] = 0.f;
    for (int q = 0; q < S - 1; ++q) issue(q);
    for (int u = 0; u < n_uses; ++u) {
      const uint32_t slot = (gu + static_cast<uint32_t>(u)) % S, par = ((gu + static_cast<uint32_t>(u)) / S) & 1u;
      fence_proxy_async();  // this thread's generic-proxy stores of the A tiles -> wgmma (async proxy) reads
      mbar_wait(smem_u32(&s_full[slot]), par);
      __syncthreads();      // the whole stage is written; the wgmma of use u - 1 have retired in both warpgroups
      const uint32_t a_hi = ring + slot * C::STAGE + static_cast<uint32_t>(wg * 8 * 128), a_lo = a_hi + C::A_TILE;
      const uint32_t b_hi = ring + slot * C::STAGE + C::A_STAGE, b_lo = b_hi + COUT * 16;  // lo rows follow the hi rows
      wg_fence();
#pragma unroll
      for (int j = 0; j < C::KC / 8; ++j) {
        const uint32_t ao = static_cast<uint32_t>(2 * j) * (kM * 16), bo = static_cast<uint32_t>(2 * j) * (2 * COUT * 16);
        const uint64_t dah = smem_desc(a_hi + ao, kM * 16, 128), dal = smem_desc(a_lo + ao, kM * 16, 128);
        const uint64_t dbh = smem_desc(b_hi + bo, 2 * COUT * 16, 128), dbl = smem_desc(b_lo + bo, 2 * COUT * 16, 128);
        wg::mma_tf32<COUT>(accx, dal, dbh, 1u);
        wg::mma_tf32<COUT>(accx, dah, dbl, 1u);
        wg::mma_tf32<COUT>(acc, dah, dbh, 1u);
      }
      wg_commit();
      issue(u + S - 1);  // the slot of use u - 1
      wg_wait<0>();
    }
    wg_fence_acc<C::ACC>(acc);
    wg_fence_acc<C::ACC>(accx);
    gu += static_cast<uint32_t>(n_uses);

    // ---------------------------------------------------------------- epilogue (accumulator fragment)
#pragma unroll
    for (int i = 0; i < C::ACC; i += 2) {
      const int r = wg * 64 + frag_row(i, wtid), c = frag_col(i, wtid);
      if (r >= rows) continue;
      float2 v = make_float2(accx[i] + acc[i], accx[i + 1] + acc[i + 1]);
      if (scale) v = make_float2(v.x * __ldg(scale + c), v.y * __ldg(scale + c + 1));
      if (shift) v = make_float2(v.x + __ldg(shift + c), v.y + __ldg(shift + c + 1));
      if (residual) {
        const float2 rv = __ldg(reinterpret_cast<const float2 *>(residual + (row0 + r) * COUT + c));
        v = make_float2(v.x + rv.x, v.y + rv.y);
      }
      if (relu) v = make_float2(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f));
      *reinterpret_cast<float2 *>(out + (row0 + r) * COUT + c) = v;
    }
  }
}

// packed[tap][g][c][hl * Cout + n][j] = split(W[tap][g*KC + 4c + j][n]): per (tap, 16-channel chunk) a K-major
// operand of 2*Cout rows (tf32 hi rows, then lo rows), so B_lo is the B_hi descriptor advanced by Cout rows.
__global__ void __launch_bounds__(256) pack_weights_kernel(const float *__restrict__ w, int K, int Cin, int Cout,
                                                           float *__restrict__ packed) {
  const long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(K) * Cin * Cout;
  if (q >= total) return;
  const int KC = kc_of(Cin), G = Cin / KC;
  const int n = static_cast<int>(q % Cout);
  const int ci = static_cast<int>((q / Cout) % Cin);
  const int t = static_cast<int>(q / (static_cast<long long>(Cout) * Cin));
  const int g = ci / KC, c = (ci % KC) / 4, j = ci & 3;
  float hi, lo;
  split_tf32(w[q], hi, lo);
  const size_t stage = static_cast<size_t>(2) * KC * Cout;  // floats per (tap, g)
  const size_t base = (static_cast<size_t>(t) * G + g) * stage + static_cast<size_t>(c) * (2 * Cout) * 4;
  packed[base + static_cast<size_t>(n) * 4 + j] = hi;
  packed[base + static_cast<size_t>(Cout + n) * 4 + j] = lo;
}

template <int CIN, int COUT>
int launch(const float *in, const int32_t *nbr, const int32_t *n_out_dev, int64_t n_cap, int K, const float *packed,
           const float *scale, const float *shift, const float *residual, int relu, float *out, cudaStream_t st,
           int splits = 1) {
  using C = Cfg<CIN, COUT>;
  const size_t smem = static_cast<size_t>(C::STAGES) * C::STAGE + static_cast<size_t>(kM) * K * sizeof(int32_t) + 1024;
  if (smem > 227 * 1024) return P3D_ERR_UNSUPPORTED;
  auto kern = gather_gemm_tf32x3_kernel<CIN, COUT>;
  P3D_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  const long long work = ((n_cap + kM - 1) / kM) * splits;
  const long long slots = static_cast<long long>(num_sms()) * C::MIN_CTAS;
  kern<<<static_cast<unsigned int>(work < slots ? work : slots), kThreads, smem, st>>>(in, nbr, n_out_dev, n_cap, K, splits, packed, scale, shift, residual, relu,
                                                  out);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

// out[r, c] = act((sum_s partial[s][r][c]) * scale + shift (+ residual)), slabs added in index order
__global__ void __launch_bounds__(256) rows_finalize_kernel(const float *__restrict__ partial, int splits,
                                                            const int32_t *__restrict__ n_dev, long long n_cap, int C,
                                                            const float *__restrict__ scale, const float *__restrict__ shift,
                                                            const float *__restrict__ residual, int relu,
                                                            float *__restrict__ out) {
  const long long n = n_dev ? min(static_cast<long long>(n_dev[0]), n_cap) : n_cap;
  const int c4 = C / 4;
  const size_t slab = static_cast<size_t>(n_cap) * C / 4;
  // persistent grid-stride loop over float4s: the grid is sized for the SMs, the trip count follows the device row count
  for (long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; q < n * c4;
       q += static_cast<long long>(gridDim.x) * blockDim.x) {
  const int c = static_cast<int>(q % c4) * 4;
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
  float r[4] = {0.f, 0.f, 0.f, 0.f};
  if (residual) {
    const float4 rv = __ldg(reinterpret_cast<const float4 *>(residual) + q);
    r[0] = rv.x;
    r[1] = rv.y;
    r[2] = rv.z;
    r[3] = rv.w;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (scale) v[j] = v[j] * __ldg(scale + c + j);
    if (shift) v[j] = v[j] + __ldg(shift + c + j);
    if (residual) v[j] = v[j] + r[j];
    if (relu) v[j] = fmaxf(v[j], 0.f);
  }
  reinterpret_cast<float4 *>(out)[q] = make_float4(v[0], v[1], v[2], v[3]);
  }
}


}  // namespace tc
}  // namespace p3d

using namespace p3d;

extern "C" size_t p3d_sparse_conv_packed_weight_bytes(int K, int Cin, int Cout) {
  if (K < 1 || Cin < 16 || Cout < 16 || Cin % 16 || Cout % 16) return 0;
  return align_up(static_cast<size_t>(K) * Cin * Cout * 2 * sizeof(float));
}

extern "C" int p3d_sparse_conv_pack_weights(const float *weight, int K, int Cin, int Cout, float *packed,
                                            p3d_stream_t stream) {
  if (!weight || !packed || K < 1) return P3D_ERR_INVALID_ARG;
  if (Cin < 16 || Cout < 16 || Cin % 16 || Cout % 16 || false) return P3D_ERR_UNSUPPORTED;
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
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // Wide layers have few 128-row tiles (52 - 130 at the C3 sizes): split the taps over 2 - 3 CTAs per tile so that all
  // SMs work on them; needs the scratch slab(s) of p3d_sparse_conv_splitk_workspace_bytes.
  int splits = tc::splits_for(Cout);
  if (splits > K) splits = K;
  const size_t need = static_cast<size_t>(splits) * static_cast<size_t>(n_out_cap) * Cout * sizeof(float);
  const bool split = splits > 1 && workspace && workspace_bytes >= need;
  float *conv_out = split ? static_cast<float *>(workspace) : out;
  const float *k_scale = split ? nullptr : scale, *k_shift = split ? nullptr : shift, *k_res = split ? nullptr : residual;
  const int k_relu = split ? 0 : relu, k_splits = split ? splits : 1;
  int rc = P3D_ERR_UNSUPPORTED;
#define P3D_TC_CASE(CI, CO)                                                                                         \
  if (Cin == CI && Cout == CO)                                                                                      \
    rc = tc::launch<CI, CO>(in, nbr, n_out_dev, n_out_cap, K, weight, k_scale, k_shift, k_res, k_relu, conv_out, st, \
                            k_splits);
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
  tc::rows_finalize_kernel<<<static_cast<unsigned int>(fin_blocks < num_sms() * 8 ? fin_blocks : num_sms() * 8), 256, 0, st>>>(conv_out, splits, n_out_dev, n_out_cap, Cout,
                                                                                scale, shift, residual, relu, out);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" int p3d_sparse_conv_gather_gemm_tf32x3(const float *in, const int32_t *nbr, const int32_t *n_out_dev,
                                                  int64_t n_out_cap, int K, int Cin, int Cout, const float *weight,
                                                  const float *scale, const float *shift, const float *residual,
                                                  int relu, float *out, p3d_stream_t stream) {
  return p3d_sparse_conv_gather_gemm_tf32x3_ws(in, nbr, n_out_dev, n_out_cap, K, Cin, Cout, weight, scale, shift, residual,
                                               relu, out, nullptr, 0, stream);
}
