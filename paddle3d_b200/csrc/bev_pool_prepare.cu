// voxel_pooling_prepare_v2 on the device (SURVEY.md §8 rows a-10 / f-3):
// LSSViewTransformer.voxel_pooling_prepare_v2, paddle3d/models/transformers/bevdet_transformer.py:230-274.
//
//   coor [B, N, D, H, W, 3] fp32 frustum points in the ego frame  ->
//   ranks_bev / ranks_depth / ranks_feat (sorted by ranks_bev), interval_starts / interval_lengths, their counts.
//
//   K1 prep_rank     per point: ((coor - lower) / interval) in fp32 (:241-242), cast toward zero (:243), range filter
//                    (:249-251), rank = b * Z*Y*X + z * Y*X + y * X + x (:256-259); points outside get the key 0xffffffff.
//   sort             stable LSD radix sort of (key, point index) over the key bits in use (cub::DeviceRadixSort, the CUDA
//                    toolkit's library sort): equal ranks keep ascending point index, which is the tie order this repo
//                    DEFINES for the reference's `argsort` (Paddle's is unspecified; the oracle uses a stable sort too).
//   K2 prep_gather   ranks_depth = index, ranks_feat = index with the depth axis removed (:235-238); first-of-run flags.
//   scan + K3        run starts compacted in order (cub::DeviceScan + scatter), lengths = next start - start (:266-271).
// The reference re-runs this (one argsort of ~500k keys in Python) every frame unless `accelerate` caches it.
//
// p3d_lss_prepare replaces K1 with lss_rank: LSSViewTransformer.get_lidar_coor (bevdet_transformer.py:147-190, PARITY
// UNPINNED) computed per frustum point in registers from a per-camera descriptor, feeding the same rank key; the sort /
// gather / scan / starts / lengths launches are shared (prep_tail).
#include <cub/cub.cuh>

#include "common.cuh"

namespace p3d {
namespace {

struct PrepGeom {
  float lo[3], iv[3];
  int gx, gy, gz;
  int D, HW;        // depth bins, H * W
  long long per_b;  // N * D * H * W points per batch sample
};

// rank key of one ego-frame point of batch sample b (:240-259); 0xffffffff = outside the grid
__device__ __forceinline__ uint32_t rank_key(const float (&pt)[3], long long b, const PrepGeom &g) {
  int c[3];
  bool ok = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float q = __fdiv_rn(__fsub_rn(pt[a], g.lo[a]), g.iv[a]);
    // cast('int64') truncates toward zero; NaN / out-of-range values can never pass the range test
    ok = ok && (q == q) && q > -2147483648.0f && q < 2147483648.0f;
    c[a] = ok ? static_cast<int>(q) : -1;
  }
  ok = ok && c[0] >= 0 && c[0] < g.gx && c[1] >= 0 && c[1] < g.gy && c[2] >= 0 && c[2] < g.gz;
  return ok ? static_cast<uint32_t>(((b * g.gz + c[2]) * g.gy + c[1]) * g.gx + c[0]) : 0xffffffffu;
}

__global__ void __launch_bounds__(256) prep_rank_kernel(const float *__restrict__ coor, long long n, PrepGeom g,
                                                        uint32_t *__restrict__ key, int32_t *__restrict__ idx) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float *p = coor + i * 3;
  const float pt[3] = {__ldg(p), __ldg(p + 1), __ldg(p + 2)};
  key[i] = rank_key(pt, i / g.per_b, g);
  idx[i] = static_cast<int32_t>(i);
}

// row r of a row-major 3x3 matrix times v, as ((m[0] * v0 + m[1] * v1) + m[2] * v2): every product and sum rounded on its
// own (no FMA contraction), so the numpy restatement in oracle/lss.py reproduces it bit for bit
__device__ __forceinline__ float row3(const float *__restrict__ m, const float (&v)[3]) {
  return __fadd_rn(__fadd_rn(__fmul_rn(__ldg(m), v[0]), __fmul_rn(__ldg(m + 1), v[1])), __fmul_rn(__ldg(m + 2), v[2]));
}

// get_lidar_coor per frustum point i = (((cam * D + d) * H + h) * W + w), cam = b * N + n, in the reference's order:
//   p = (x[w], y[h], depth[d]) - post_trans;  q = inv(post_rots) . p;  s = (q0 * q2, q1 * q2, q2);
//   e = combine . s + sensor2ego[:3, 3]  (the translation added after the row sum);  o = bda . e
// then the rank key of o.  coor (nullable) receives o as [B, N, D, H, W, 3].
__global__ void __launch_bounds__(256) lss_rank_kernel(const p3d_lss_camera *__restrict__ cams, const float *__restrict__ bda,
                                                       const float *__restrict__ axis_d, const float *__restrict__ axis_x,
                                                       const float *__restrict__ axis_y, long long n, PrepGeom g, int N, int H,
                                                       int W, float *__restrict__ coor, uint32_t *__restrict__ key,
                                                       int32_t *__restrict__ idx) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int j = static_cast<int>(i);  // n <= 2^31 - 1: 32-bit index arithmetic
  const int w = j % W, t = j / W;
  const int h = t % H, cd = t / H;  // cd = cam * D + d
  const int d = cd % g.D, cam = cd / g.D;
  const long long b = cam / N;
  const p3d_lss_camera *c = cams + cam;
  const float p[3] = {__fsub_rn(__ldg(axis_x + w), __ldg(c->post_trans)), __fsub_rn(__ldg(axis_y + h), __ldg(c->post_trans + 1)),
                      __fsub_rn(__ldg(axis_d + d), __ldg(c->post_trans + 2))};
  const float q[3] = {row3(c->inv_post_rot, p), row3(c->inv_post_rot + 3, p), row3(c->inv_post_rot + 6, p)};
  const float s[3] = {__fmul_rn(q[0], q[2]), __fmul_rn(q[1], q[2]), q[2]};
  const float e[3] = {__fadd_rn(row3(c->combine, s), __ldg(c->trans)), __fadd_rn(row3(c->combine + 3, s), __ldg(c->trans + 1)),
                      __fadd_rn(row3(c->combine + 6, s), __ldg(c->trans + 2))};
  const float *m = bda + b * 9;
  const float o[3] = {row3(m, e), row3(m + 3, e), row3(m + 6, e)};
  if (coor) {
    coor[i * 3] = o[0];
    coor[i * 3 + 1] = o[1];
    coor[i * 3 + 2] = o[2];
  }
  key[i] = rank_key(o, b, g);
  idx[i] = static_cast<int32_t>(i);
}

__global__ void __launch_bounds__(256) prep_gather_kernel(const uint32_t *__restrict__ key_sorted,
                                                          const int32_t *__restrict__ idx_sorted, long long n, PrepGeom g,
                                                          int32_t *__restrict__ ranks_bev, int32_t *__restrict__ ranks_depth,
                                                          int32_t *__restrict__ ranks_feat, int32_t *__restrict__ flag,
                                                          int32_t *__restrict__ counts) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t k = key_sorted[i];
  const bool kept = k != 0xffffffffu;
  const int32_t p = idx_sorted[i];
  ranks_bev[i] = kept ? static_cast<int32_t>(k) : 0;
  ranks_depth[i] = kept ? p : 0;
  // index into [B, N, H, W] features: drop the depth axis of the [B, N, D, H, W] point index
  const long long cam = p / (static_cast<long long>(g.D) * g.HW);
  ranks_feat[i] = kept ? static_cast<int32_t>(cam * g.HW + p % g.HW) : 0;
  const bool first = kept && (i == 0 || key_sorted[i - 1] != k);
  flag[i] = first ? 1 : 0;
  if (kept && (i == n - 1 || key_sorted[i + 1] == 0xffffffffu)) counts[0] = static_cast<int32_t>(i + 1);  // n_kept
  if (i == 0 && !kept) counts[0] = 0;
}

__global__ void __launch_bounds__(256) prep_starts_kernel(const int32_t *__restrict__ flag, const int32_t *__restrict__ pos,
                                                          long long n, int32_t *__restrict__ starts,
                                                          int32_t *__restrict__ counts) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (flag[i]) starts[pos[i]] = static_cast<int32_t>(i);
  if (i == n - 1) counts[1] = pos[i] + flag[i];  // n_intervals
}

__global__ void __launch_bounds__(256) prep_lengths_kernel(const int32_t *__restrict__ starts, const int32_t *__restrict__ counts,
                                                           long long n, int32_t *__restrict__ lengths) {
  const long long j = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int n_int = counts[1], n_kept = counts[0];
  if (j >= n) return;
  if (j < n_int) {
    lengths[j] = (j + 1 < n_int ? starts[j + 1] : n_kept) - starts[j];
  } else {
    lengths[j] = 0;
  }
}

struct PrepWs {
  uint32_t *key, *key_sorted;
  int32_t *idx, *idx_sorted, *flag, *pos;
  void *cub_tmp;
  size_t cub_bytes, bytes;
};

PrepWs carve(void *ws, long long n, int key_bits) {
  PrepWs w;
  Carver c(ws);
  const size_t m = static_cast<size_t>(n > 0 ? n : 1);
  w.key = c.take<uint32_t>(m);
  w.key_sorted = c.take<uint32_t>(m);
  w.idx = c.take<int32_t>(m);
  w.idx_sorted = c.take<int32_t>(m);
  w.flag = c.take<int32_t>(m);
  w.pos = c.take<int32_t>(m);
  size_t a = 0, b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, a, static_cast<const uint32_t *>(nullptr), static_cast<uint32_t *>(nullptr),
                                  static_cast<const int32_t *>(nullptr), static_cast<int32_t *>(nullptr), static_cast<int>(m), 0,
                                  key_bits);
  cub::DeviceScan::ExclusiveSum(nullptr, b, static_cast<const int32_t *>(nullptr), static_cast<int32_t *>(nullptr),
                                static_cast<int>(m));
  w.cub_bytes = a > b ? a : b;
  w.cub_tmp = c.take<char>(w.cub_bytes);
  w.bytes = c.off;
  return w;
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" size_t p3d_bev_pool_prepare_workspace_bytes(int64_t num_points) {
  if (num_points < 0 || num_points > 0x7fffffffll) return 0;
  return carve(nullptr, num_points, 32).bytes;
}

namespace p3d {
namespace {

// Argument checks shared by both entry points (status codes before any CUDA call), then the geometry and workspace carve.
int prep_setup(int B, int N, int D, int H, int W, const float *lower, const float *interval, const int32_t *grid_size,
               const void *const *outs, void *workspace, size_t workspace_bytes, PrepGeom *g, PrepWs *w, long long *n_out) {
  for (int k = 0; k < 6; ++k)
    if (!outs[k]) return P3D_ERR_INVALID_ARG;
  if (!lower || !interval || !grid_size || !workspace || B < 1 || N < 1 || D < 1 || H < 1 || W < 1) return P3D_ERR_INVALID_ARG;
  const long long n = static_cast<long long>(B) * N * D * H * W;
  const long long cells = static_cast<long long>(B) * grid_size[0] * grid_size[1] * grid_size[2];
  // ranks are int32: the largest, cells - 1, must fit (a larger key would be stored as a negative rank)
  if (n > 0x7fffffffll || cells < 1 || cells > 0x80000000ll || grid_size[0] < 1 || grid_size[1] < 1 || grid_size[2] < 1)
    return P3D_ERR_UNSUPPORTED;
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return P3D_ERR_INVALID_ARG;
  for (int a = 0; a < 3; ++a) {
    g->lo[a] = lower[a];
    g->iv[a] = interval[a];
  }
  g->gx = grid_size[0];
  g->gy = grid_size[1];
  g->gz = grid_size[2];
  g->D = D;
  g->HW = H * W;
  g->per_b = static_cast<long long>(N) * D * H * W;
  *w = carve(workspace, n, 32);
  if (workspace_bytes < w->bytes) return P3D_ERR_WORKSPACE;
  *n_out = n;
  return P3D_OK;
}

// Everything after the keys: sort, gather, scan, starts, lengths.
int prep_tail(const PrepWs &w, long long n, const PrepGeom &g, int32_t *ranks_bev, int32_t *ranks_depth, int32_t *ranks_feat,
              int32_t *interval_starts, int32_t *interval_lengths, int32_t *counts_dev, cudaStream_t st) {
  const unsigned int blocks = div_up(n, 256);
  size_t tmp = w.cub_bytes;
  // all 32 key bits: the invalid key 0xffffffff must sort behind every cell rank
  P3D_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(w.cub_tmp, tmp, w.key, w.key_sorted, w.idx, w.idx_sorted, static_cast<int>(n), 0,
                                                 32, st));
  P3D_CUDA_CHECK(cudaMemsetAsync(counts_dev, 0, 2 * sizeof(int32_t), st));
  prep_gather_kernel<<<blocks, 256, 0, st>>>(w.key_sorted, w.idx_sorted, n, g, ranks_bev, ranks_depth, ranks_feat, w.flag,
                                             counts_dev);
  P3D_LAUNCH_CHECK();
  tmp = w.cub_bytes;
  P3D_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(w.cub_tmp, tmp, w.flag, w.pos, static_cast<int>(n), st));
  prep_starts_kernel<<<blocks, 256, 0, st>>>(w.flag, w.pos, n, interval_starts, counts_dev);
  P3D_LAUNCH_CHECK();
  prep_lengths_kernel<<<blocks, 256, 0, st>>>(interval_starts, counts_dev, n, interval_lengths);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

}  // namespace
}  // namespace p3d

extern "C" int p3d_bev_pool_prepare(const float *coor, int B, int N, int D, int H, int W, const float *grid_lower_bound_host,
                                    const float *grid_interval_host, const int32_t *grid_size_host, int32_t *ranks_bev,
                                    int32_t *ranks_depth, int32_t *ranks_feat, int32_t *interval_starts,
                                    int32_t *interval_lengths, int32_t *counts_dev, void *workspace, size_t workspace_bytes,
                                    p3d_stream_t stream) {
  if (!coor) return P3D_ERR_INVALID_ARG;
  const void *outs[6] = {ranks_bev, ranks_depth, ranks_feat, interval_starts, interval_lengths, counts_dev};
  PrepGeom g;
  PrepWs w;
  long long n = 0;
  const int rc = prep_setup(B, N, D, H, W, grid_lower_bound_host, grid_interval_host, grid_size_host, outs, workspace,
                            workspace_bytes, &g, &w, &n);
  if (rc != P3D_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  prep_rank_kernel<<<div_up(n, 256), 256, 0, st>>>(coor, n, g, w.key, w.idx);
  P3D_LAUNCH_CHECK();
  return prep_tail(w, n, g, ranks_bev, ranks_depth, ranks_feat, interval_starts, interval_lengths, counts_dev, st);
}

extern "C" int p3d_lss_prepare(const p3d_lss_camera *cams, const float *bda, const float *axis_depth, const float *axis_x,
                               const float *axis_y, int B, int N, int D, int H, int W, const float *grid_lower_bound_host,
                               const float *grid_interval_host, const int32_t *grid_size_host, float *coor,
                               int32_t *ranks_bev, int32_t *ranks_depth, int32_t *ranks_feat, int32_t *interval_starts,
                               int32_t *interval_lengths, int32_t *counts_dev, void *workspace, size_t workspace_bytes,
                               p3d_stream_t stream) {
  if (!cams || !bda || !axis_depth || !axis_x || !axis_y) return P3D_ERR_INVALID_ARG;
  const void *outs[6] = {ranks_bev, ranks_depth, ranks_feat, interval_starts, interval_lengths, counts_dev};
  PrepGeom g;
  PrepWs w;
  long long n = 0;
  const int rc = prep_setup(B, N, D, H, W, grid_lower_bound_host, grid_interval_host, grid_size_host, outs, workspace,
                            workspace_bytes, &g, &w, &n);
  if (rc != P3D_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  lss_rank_kernel<<<div_up(n, 256), 256, 0, st>>>(cams, bda, axis_depth, axis_x, axis_y, n, g, N, H, W, coor, w.key, w.idx);
  P3D_LAUNCH_CHECK();
  return prep_tail(w, n, g, ranks_bev, ranks_depth, ranks_feat, interval_starts, interval_lengths, counts_dev, st);
}
