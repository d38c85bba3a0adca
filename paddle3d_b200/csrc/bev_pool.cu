// bev_pool_v2 forward / backward for sm_90a.
//
// Replaces paddle3d/ops/bev_pool_v2/bev_pool_cuda.cu:18-116 (and the duplicate in
// ops/bev_pool_v2_backward).  Same arithmetic in the same order — one fp32 FMA per point, summed in
// index order, so results are bit-identical to the reference kernels — but
//   * a thread owns 4 channels (float4 feature loads, 16 B stores) instead of one, so the rank /
//     depth words are fetched once per 4 channels and the feature row of a point is read as
//     contiguous 16 B pieces by adjacent lanes;
//   * launched on the caller's stream (the reference uses the default stream, .cu:102);
//   * the zero fill of the output is an async memset on the same stream.
// Algorithmic bytes: 12*n_pts ranks + 4*n_pts depth + 4*|feat| + 8*n_int + 4*|out|.
#include <stdlib.h>

#include "common.cuh"
#include "h16.cuh"

namespace p3d {
namespace {

template <int V>
struct Vec;
template <>
struct Vec<4> {
  using T = float4;
};
template <>
struct Vec<1> {
  using T = float;
};

template <int V>
__global__ void __launch_bounds__(256) bev_fwd_kernel(int cv, int n_intervals, const float *__restrict__ depth,
                                                      const float *__restrict__ feat,
                                                      const int *__restrict__ ranks_depth,
                                                      const int *__restrict__ ranks_feat,
                                                      const int *__restrict__ ranks_bev,
                                                      const int *__restrict__ interval_starts,
                                                      const int *__restrict__ interval_lengths,
                                                      float *__restrict__ out) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int k = static_cast<int>(idx / cv);
  const int j = static_cast<int>(idx - static_cast<long long>(k) * cv);
  if (k >= n_intervals) return;
  const int s = interval_starts[k], len = interval_lengths[k];
  const int c = cv * V;
  float acc[V];
#pragma unroll
  for (int v = 0; v < V; ++v) acc[v] = 0.f;
#pragma unroll 4
  for (int i = 0; i < len; ++i) {
    const float d = __ldg(depth + ranks_depth[s + i]);
    const float *f = feat + static_cast<size_t>(ranks_feat[s + i]) * c + j * V;
    if (V == 4) {
      const float4 fv = __ldg(reinterpret_cast<const float4 *>(f));
      acc[0] = fmaf(fv.x, d, acc[0]);
      acc[1] = fmaf(fv.y, d, acc[1]);
      acc[2] = fmaf(fv.z, d, acc[2]);
      acc[3] = fmaf(fv.w, d, acc[3]);
    } else {
      acc[0] = fmaf(__ldg(f), d, acc[0]);
    }
  }
  float *o = out + static_cast<size_t>(ranks_bev[s]) * c + j * V;
  if (V == 4)
    *reinterpret_cast<float4 *>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
  else
    o[0] = acc[0];
}

// Forward, redesigned (round 2): ONE WARP PER INTERVAL.  The reference kernel (and the round-1 float4 variant above, kept
// for channel counts that are not a multiple of 4) gives every (interval, channel) its own thread, so each of them walks
// the interval's rank / depth words again and sits on one dependent load -> FMA chain; the long near-camera intervals
// (thousands of points in one cell) then set the kernel time.  Here the 32 lanes fetch the rank and depth words of 32
// consecutive points ONCE (three coalesced loads + one gather), broadcast them by shuffle, every lane owns up to two
// float4 channel groups (C <= 256), and the feature rows of the next 8 points are in flight while the current ones are
// accumulated.  Per channel the fp32 FMA chain runs over the points in index order, exactly as bev_pool_cuda.cu:24-43:
// results stay bit-identical to the reference kernel.
// DEV: the interval count is read from counts_dev[1] (the grid covers an upper bound; warps at or past the count exit), so
// one captured graph serves every calibration.  PLANAR: the output is [B, Z * C, Y, X] with channel z * C + c, the layout
// view_transform returns (torch.cat(bev.unbind(dim=2), 1) of the [B, C, Z, Y, X] pool), instead of [B, Z, Y, X, C];
// yx = Y * X.  PIX: the output is pixel H16 rows [B, Y, X, row_c] (the image the dense fp16-pair convs read), channel
// z * C + c of the planar layout at row b * Y*X + y * X + x, split into (hi, lo'); Z = cells along z.  The accumulation is
// the same in every instantiation.
template <int G, bool DEV = false, bool PLANAR = false, bool PIX = false>
__global__ void __launch_bounds__(256) bev_fwd_warp_kernel(int cv, int n_intervals, const float *__restrict__ depth,
                                                           const float *__restrict__ feat,
                                                           const int *__restrict__ ranks_depth,
                                                           const int *__restrict__ ranks_feat,
                                                           const int *__restrict__ ranks_bev,
                                                           const int *__restrict__ interval_starts,
                                                           const int *__restrict__ interval_lengths,
                                                           float *__restrict__ out, const int *__restrict__ counts_dev = nullptr,
                                                           int yx = 0, int Z = 1, int row_c = 0, int32_t *status = nullptr) {
  const int k = static_cast<int>((static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (k >= (DEV ? __ldg(counts_dev + 1) : n_intervals)) return;
  const int s = interval_starts[k], len = interval_lengths[k];
  const int c = cv * 4;
  bool own[G];
  float4 acc[G];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    own[g] = lane + 32 * g < cv;
    acc[g] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  constexpr int U = (G == 1) ? 16 : 8;  // feature rows in flight per lane
  // three-deep software pipeline over batches of 32 points, so that a long interval pays each memory round trip once per
  // batch instead of three dependent ones: rank words of batch b + 2, depth gather of batch b + 1, features of batch b
  int rf_cur = 0, rf_nxt = 0, rd_nxt = 0;
  float d_cur = 0.f;
  if (lane < len) {
    rf_cur = __ldg(ranks_feat + s + lane);
    d_cur = __ldg(depth + __ldg(ranks_depth + s + lane));
  }
  if (32 + lane < len) {
    rf_nxt = __ldg(ranks_feat + s + 32 + lane);
    rd_nxt = __ldg(ranks_depth + s + 32 + lane);
  }
  for (int base = 0; base < len; base += 32) {
    const int m = min(32, len - base);
    float d_nxt = 0.f;
    int rf_nn = 0, rd_nn = 0;
    if (base + 32 + lane < len) d_nxt = __ldg(depth + rd_nxt);
    if (base + 64 + lane < len) {
      rf_nn = __ldg(ranks_feat + s + base + 64 + lane);
      rd_nn = __ldg(ranks_depth + s + base + 64 + lane);
    }
    for (int i0 = 0; i0 < m; i0 += U) {
      float4 f[U][G];
      float d[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = i0 + u < m ? i0 + u : m - 1;  // clamp: the shuffles stay warp-uniform, the extra loads are discarded
        const int rf = __shfl_sync(0xffffffffu, rf_cur, i);
        d[u] = __shfl_sync(0xffffffffu, d_cur, i);
#pragma unroll
        for (int g = 0; g < G; ++g)
          if (own[g]) f[u][g] = __ldg(reinterpret_cast<const float4 *>(feat + static_cast<size_t>(rf) * c) + lane + 32 * g);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (i0 + u < m) {
#pragma unroll
          for (int g = 0; g < G; ++g)
            if (own[g]) {
              acc[g].x = fmaf(f[u][g].x, d[u], acc[g].x);
              acc[g].y = fmaf(f[u][g].y, d[u], acc[g].y);
              acc[g].z = fmaf(f[u][g].z, d[u], acc[g].z);
              acc[g].w = fmaf(f[u][g].w, d[u], acc[g].w);
            }
        }
      }
    }
    rf_cur = rf_nxt;
    d_cur = d_nxt;
    rf_nxt = rf_nn;
    rd_nxt = rd_nn;
  }
  if (PIX) {
    // rank b * Z*Y*X + z * Y*X + (y * X + x): row b * Y*X + y * X + x, channels z * C + 4 (lane + 32 g) .. + 3, whose hi
    // halves are 8 bytes at (ch / 32) * 128 + (ch % 32) * 2 of the row and the lo' halves 64 bytes further
    const int rb = __ldg(ranks_bev + s), bz = rb / yx;
    uint8_t *row = reinterpret_cast<uint8_t *>(out) + (static_cast<size_t>(bz / Z) * yx + rb % yx) * (4 * static_cast<size_t>(row_c));
    bool ovf = false;
#pragma unroll
    for (int g = 0; g < G; ++g)
      if (own[g]) {
        const int ch = (bz % Z) * c + 4 * (lane + 32 * g);
        __half2 h01, l01, h23, l23;
        split_h16x2(acc[g].x, acc[g].y, h01, l01, ovf);
        split_h16x2(acc[g].z, acc[g].w, h23, l23, ovf);
        uint8_t *o = row + (ch >> 5) * 128 + (ch & 31) * 2;
        *reinterpret_cast<uint2 *>(o) = make_uint2(*reinterpret_cast<const uint32_t *>(&h01), *reinterpret_cast<const uint32_t *>(&h23));
        *reinterpret_cast<uint2 *>(o + 64) = make_uint2(*reinterpret_cast<const uint32_t *>(&l01), *reinterpret_cast<const uint32_t *>(&l23));
      }
    if (ovf && status) atomicOr(status, 1);
    return;
  }
  if (PLANAR) {
    const int rb = __ldg(ranks_bev + s);  // b * Z*Y*X + z * Y*X + (y * X + x): plane (b * Z + z) * C + c
    float *o = out + static_cast<size_t>(rb / yx) * c * yx + rb % yx;
#pragma unroll
    for (int g = 0; g < G; ++g)
      if (own[g]) {
        const size_t ch = 4 * (lane + 32 * g);
        o[ch * yx] = acc[g].x;
        o[(ch + 1) * yx] = acc[g].y;
        o[(ch + 2) * yx] = acc[g].z;
        o[(ch + 3) * yx] = acc[g].w;
      }
    return;
  }
  float4 *o = reinterpret_cast<float4 *>(out + static_cast<size_t>(__ldg(ranks_bev + s)) * c);
#pragma unroll
  for (int g = 0; g < G; ++g)
    if (own[g]) o[lane + 32 * g] = acc[g];
}

// One warp per interval.  Phase 1: lanes stride over the interval's points, each doing the
// sequential dot product over channels (depth_grad).  Phase 2: lanes stride over channels, each
// doing the sequential sum over the interval's points (feat_grad).  Orders match .cu:62-94.
__global__ void __launch_bounds__(256) bev_bwd_kernel(int c, int n_intervals, const float *__restrict__ out_grad,
                                                      const float *__restrict__ depth, const float *__restrict__ feat,
                                                      const int *__restrict__ ranks_depth,
                                                      const int *__restrict__ ranks_feat,
                                                      const int *__restrict__ ranks_bev,
                                                      const int *__restrict__ interval_starts,
                                                      const int *__restrict__ interval_lengths,
                                                      float *__restrict__ depth_grad, float *__restrict__ feat_grad) {
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (k >= n_intervals) return;
  const int s = interval_starts[k], len = interval_lengths[k];
  for (int i = lane; i < len; i += 32) {
    const float *og = out_grad + static_cast<size_t>(ranks_bev[s + i]) * c;
    const float *ff = feat + static_cast<size_t>(ranks_feat[s + i]) * c;
    float g = 0.f;
    for (int cc = 0; cc < c; ++cc) g = fmaf(__ldg(og + cc), __ldg(ff + cc), g);
    depth_grad[ranks_depth[s + i]] = g;
  }
  float *fg = feat_grad + static_cast<size_t>(ranks_feat[s]) * c;
  for (int cc = lane; cc < c; cc += 32) {
    float g = 0.f;
    for (int i = 0; i < len; ++i)
      g = fmaf(__ldg(out_grad + static_cast<size_t>(ranks_bev[s + i]) * c + cc), __ldg(depth + ranks_depth[s + i]), g);
    fg[cc] = g;
  }
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_bev_pool_v2(const float *depth, const float *feat, const int32_t *ranks_depth,
                               const int32_t *ranks_feat, const int32_t *ranks_bev, const int32_t *interval_lengths,
                               const int32_t *interval_starts, int n_intervals, int c, float *out,
                               int64_t out_numel, p3d_stream_t stream) {
  if (n_intervals < 0 || c < 1 || out_numel < 0 || !out) return P3D_ERR_INVALID_ARG;
  if (n_intervals && (!depth || !feat || !ranks_depth || !ranks_feat || !ranks_bev || !interval_lengths ||
                      !interval_starts))
    return P3D_ERR_INVALID_ARG;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  P3D_CUDA_CHECK(cudaMemsetAsync(out, 0, static_cast<size_t>(out_numel) * sizeof(float), st));  // bev_pool.cc:47-48
  if (n_intervals == 0) return P3D_OK;
  const bool vec = (c % 4 == 0) && !(reinterpret_cast<uintptr_t>(feat) & 15) && !(reinterpret_cast<uintptr_t>(out) & 15);
  static const int variant = getenv("P3D_BEV_POOL_VARIANT") ? atoi(getenv("P3D_BEV_POOL_VARIANT")) : 0;  // 1: round-1 kernel
  if (vec && c <= 256 && variant == 0) {
    const int cv = c / 4;
    const unsigned int blocks = div_up(static_cast<long long>(n_intervals) * 32, 256);
    if (cv <= 32)
      bev_fwd_warp_kernel<1><<<blocks, 256, 0, st>>>(cv, n_intervals, depth, feat, ranks_depth, ranks_feat, ranks_bev,
                                                     interval_starts, interval_lengths, out);
    else
      bev_fwd_warp_kernel<2><<<blocks, 256, 0, st>>>(cv, n_intervals, depth, feat, ranks_depth, ranks_feat, ranks_bev,
                                                     interval_starts, interval_lengths, out);
  } else if (vec) {
    const int cv = c / 4;
    bev_fwd_kernel<4><<<div_up(static_cast<long long>(n_intervals) * cv, 256), 256, 0, st>>>(
        cv, n_intervals, depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths, out);
  } else {
    bev_fwd_kernel<1><<<div_up(static_cast<long long>(n_intervals) * c, 256), 256, 0, st>>>(
        c, n_intervals, depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths, out);
  }
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" int p3d_bev_pool_v2_dev(const float *depth, const float *feat, const int32_t *ranks_depth,
                                   const int32_t *ranks_feat, const int32_t *ranks_bev, const int32_t *interval_lengths,
                                   const int32_t *interval_starts, const int32_t *counts_dev, int64_t capacity, int c, int B,
                                   int Z, int Y, int X, int planar, float *out, p3d_stream_t stream) {
  if (!depth || !feat || !ranks_depth || !ranks_feat || !ranks_bev || !interval_lengths || !interval_starts || !counts_dev ||
      !out || capacity < 0 || c < 1 || B < 1 || Z < 1 || Y < 1 || X < 1 || (planar != 0 && planar != 1))
    return P3D_ERR_INVALID_ARG;
  const long long cells = static_cast<long long>(B) * Z * Y * X;  // <= 2^31: every rank, at most cells - 1, is an int32
  if (c % 4 || c > 256 || (reinterpret_cast<uintptr_t>(feat) & 15) || (reinterpret_cast<uintptr_t>(out) & 15) ||
      capacity > 0x7fffffffll || cells > 0x80000000ll || static_cast<long long>(Y) * X > 0x7fffffffll)
    return P3D_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  P3D_CUDA_CHECK(cudaMemsetAsync(out, 0, static_cast<size_t>(cells) * c * sizeof(float), st));
  // every interval is a distinct cell: the count is bounded by the cells as well as by the rank capacity
  const long long bound = capacity < cells ? capacity : cells;
  if (bound == 0) return P3D_OK;
  const int cv = c / 4, yx = Y * X;
  const unsigned int blocks = div_up(bound * 32, 256);
  const int n = static_cast<int>(bound);
#define P3D_BEV_DEV(G, P)                                                                                                  \
  bev_fwd_warp_kernel<G, true, P><<<blocks, 256, 0, st>>>(cv, n, depth, feat, ranks_depth, ranks_feat, ranks_bev,         \
                                                          interval_starts, interval_lengths, out, counts_dev, yx)
  if (cv <= 32) {
    if (planar) P3D_BEV_DEV(1, true); else P3D_BEV_DEV(1, false);
  } else {
    if (planar) P3D_BEV_DEV(2, true); else P3D_BEV_DEV(2, false);
  }
#undef P3D_BEV_DEV
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" int p3d_bev_pool_v2_dev_h16(const float *depth, const float *feat, const int32_t *ranks_depth,
                                       const int32_t *ranks_feat, const int32_t *ranks_bev, const int32_t *interval_lengths,
                                       const int32_t *interval_starts, const int32_t *counts_dev, int64_t capacity, int c,
                                       int B, int Z, int Y, int X, void *out_h16, int out_C, int32_t *status_dev,
                                       p3d_stream_t stream) {
  if (!depth || !feat || !ranks_depth || !ranks_feat || !ranks_bev || !interval_lengths || !interval_starts || !counts_dev ||
      !out_h16 || capacity < 0 || c < 1 || B < 1 || Z < 1 || Y < 1 || X < 1 || out_C < 32 || out_C % 32 ||
      static_cast<long long>(Z) * c > out_C)
    return P3D_ERR_INVALID_ARG;
  const long long cells = static_cast<long long>(B) * Z * Y * X;
  if (c % 4 || c > 256 || (reinterpret_cast<uintptr_t>(feat) & 15) || (reinterpret_cast<uintptr_t>(out_h16) & 15) ||
      capacity > 0x7fffffffll || cells > 0x80000000ll || static_cast<long long>(Y) * X > 0x7fffffffll)
    return P3D_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // empty cells and the channels from Z * c up to out_C stay zero
  P3D_CUDA_CHECK(cudaMemsetAsync(out_h16, 0, static_cast<size_t>(B) * Y * X * out_C * 4, st));
  const long long bound = capacity < cells ? capacity : cells;
  if (bound == 0) return P3D_OK;
  const int cv = c / 4, yx = Y * X;
  const unsigned int blocks = div_up(bound * 32, 256);
  const int n = static_cast<int>(bound);
  // one instantiation for every c: G = 2 keeps 8 feature rows in flight per lane, which fits the registers without
  // spilling (G = 1's 16 do not once the split is added); lanes past c / 4 only take part in the shuffles
  bev_fwd_warp_kernel<2, true, false, true><<<blocks, 256, 0, st>>>(cv, n, depth, feat, ranks_depth, ranks_feat, ranks_bev,
                                                                   interval_starts, interval_lengths, static_cast<float *>(out_h16),
                                                                   counts_dev, yx, Z, out_C, status_dev);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" int p3d_bev_pool_v2_bkwd(const float *out_grad, const float *depth, const float *feat,
                                    const int32_t *ranks_depth, const int32_t *ranks_feat, const int32_t *ranks_bev,
                                    const int32_t *interval_lengths, const int32_t *interval_starts, int n_intervals,
                                    int c, float *depth_grad, int64_t depth_numel, float *feat_grad,
                                    int64_t feat_numel, p3d_stream_t stream) {
  if (n_intervals < 0 || c < 1 || depth_numel < 0 || feat_numel < 0 || !depth_grad || !feat_grad)
    return P3D_ERR_INVALID_ARG;
  if (n_intervals && (!out_grad || !depth || !feat || !ranks_depth || !ranks_feat || !ranks_bev ||
                      !interval_lengths || !interval_starts))
    return P3D_ERR_INVALID_ARG;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  P3D_CUDA_CHECK(cudaMemsetAsync(depth_grad, 0, static_cast<size_t>(depth_numel) * sizeof(float), st));
  P3D_CUDA_CHECK(cudaMemsetAsync(feat_grad, 0, static_cast<size_t>(feat_numel) * sizeof(float), st));
  if (n_intervals == 0) return P3D_OK;
  bev_bwd_kernel<<<div_up(static_cast<long long>(n_intervals) * 32, 256), 256, 0, st>>>(
      c, n_intervals, out_grad, depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths,
      depth_grad, feat_grad);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
