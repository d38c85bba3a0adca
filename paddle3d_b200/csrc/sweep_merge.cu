// merge_sweeps for sm_90a: the multi-sweep input of the nuScenes 10-sweep CenterPoint model, on the device.
//
// Replaces the host-side merge of LoadPointCloud.__call__ (paddle3d/transforms/reader.py:116-167; restated in numpy by
// paddle3d_b200/io.py merge_sweeps): key rows, then each earlier sweep's rows outside the |x|, |y| < r square, moved into
// the key frame by ref_from_curr (fp64, rounded once to fp32), with a time-lag column.  The output ROW ORDER is the
// reference's concatenation order: hard_voxelize numbers voxels by first appearance and keeps the first P points of each
// voxel, so the order decides the voxels.
//
//   K1 merge_sweeps  one pass over the virtual concatenation of all entries, in tiles of 1024 rows (an entry's rows are
//                    cut into a fixed number of tiles, so one grid size serves every frame of a captured graph).  A tile
//                    stages its raw rows in shared memory with 16-byte loads, computes the keep flags, ranks the kept
//                    rows with warp ballots + one warp scan, gets its output offset by decoupled look-back across tiles
//                    (common.cuh, shared with hard_voxelize's rank kernel), builds its output rows in shared memory and
//                    streams them out as 16-byte stores.
//   K2 merge_tail    (PDL) NaN rows from n_out to cap - hard_voxelize drops them - and the status word.
//
// The frustum instantiation (p3d_merge_sweeps_frustum, one entry) is the KITTI camera cull of Paddle3D's
// RemoveCameraInvisiblePointsKITTI / SECOND's remove_outside_points: the keep stage also tests each row against six
// planes read from the device on every launch (one captured graph serves every calibration and image size), in the
// reference's fp64 arithmetic, unfused; paddle3d_b200/kitti.py remove_camera_invisible is its oracle.
//
// Bandwidth-bound: 4 * raw_dim * rows bytes read, 4 * F * cap bytes written.
#include <math.h>

#include "common.cuh"

namespace p3d {
namespace {

constexpr int kMergeBlock = 256;
constexpr int kMergeItems = 4;                         // rows per thread: row k * 256 + tid of the tile
constexpr int kMergeTile = kMergeBlock * kMergeItems;  // rows per tile
constexpr int kMergeWarps = kMergeBlock / 32;
constexpr int kMaxCols = 11;  // raw_dim + F: both staging tiles fit 44 KB of shared memory
static_assert(kMergeItems * kMergeWarps == 32, "one warp scans the (item, warp) counts");

struct MergeAttrs {
  int raw_dim, F, ncol, use_time_lag;
  int col[kMaxCols];  // selected raw columns
  float radius;
};

struct MergeWs {
  unsigned long long *scan;  // [1 + tiles]: ticket, then the look-back descriptors
  int32_t *flags;            // status bits gathered during the pass
  size_t bytes;
};

MergeWs carve_merge(void *ws, long long tiles) {
  MergeWs w;
  Carver c(ws);
  w.scan = c.take<unsigned long long>(static_cast<size_t>(tiles) + 1);
  w.flags = c.take<int32_t>(1);
  w.bytes = c.off;
  return w;
}

template <bool kFrustum>
__global__ void __launch_bounds__(kMergeBlock) merge_sweeps_kernel(const float *__restrict__ raw, int num_slots,
                                                                   long long slot_cap,
                                                                   const p3d_sweep_desc *__restrict__ desc,
                                                                   int tiles_per_entry, MergeAttrs a,
                                                                   float *__restrict__ out, long long cap,
                                                                   unsigned long long *__restrict__ scan,
                                                                   int32_t *__restrict__ flags,
                                                                   int32_t *__restrict__ n_out,
                                                                   const double *__restrict__ planes) {
  extern __shared__ __align__(16) float s_mem[];
  __shared__ double s_m[12];
  __shared__ double s_pl[kFrustum ? 24 : 1];  // frustum: six (a, b, c, d) planes, outward normals
  __shared__ int s_col[kMaxCols];
  __shared__ int s_cnt[kMergeItems * kMergeWarps];
  __shared__ unsigned int s_bid;
  __shared__ int s_entry, s_nr, s_tf, s_prefix, s_agg;
  __shared__ float s_lag;
  __shared__ long long s_src;
  pdl_trigger();
  pdl_wait();
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int RD = a.raw_dim, F = a.F;
  float *s_in = s_mem;                  // [kMergeTile][raw_dim]
  float *s_out = s_mem + kMergeTile * RD;  // [kMergeTile][F]
  if (tid < a.ncol) s_col[tid] = a.col[tid];
  if (tid == 0) {
    const unsigned int bid = static_cast<unsigned int>(atomicAdd(&scan[0], 1ull));
    const int e = static_cast<int>(bid / tiles_per_entry), t = static_cast<int>(bid % tiles_per_entry);
    const p3d_sweep_desc *d = desc + e;
    const int slot = d->slot, rows = d->rows;
    const bool bad = slot < 0 || slot >= num_slots || rows < 0 || rows > slot_cap;
    if (bad && t == 0) atomicOr(flags, 2);
    const long long r0 = static_cast<long long>(t) * kMergeTile;
    const long long left = bad ? 0 : rows - r0;
    s_bid = bid;
    s_entry = e;
    s_nr = static_cast<int>(left < 0 ? 0 : (left > kMergeTile ? kMergeTile : left));
    s_tf = e > 0 && d->has_transform;  // the key sweep is never moved and carries lag 0
    s_lag = e > 0 ? d->time_lag : 0.f;
    s_src = bad ? 0 : (static_cast<long long>(slot) * slot_cap + r0) * RD;
  }
  __syncthreads();
  const int e = s_entry, nr = s_nr;
  if (tid < 12) s_m[tid] = desc[e].ref_from_curr[tid];  // read after the next barrier
  if (kFrustum && tid < 24) s_pl[tid] = planes[tid];
  // stage the tile's raw rows: 16-byte loads (slot_cap % 4 == 0, tiles start at multiples of 1024 rows)
  if (nr > 0) {
    const float *src = raw + s_src;
    const int nf = nr * RD, n4 = nf >> 2;
    for (int q = tid; q < n4; q += kMergeBlock)
      reinterpret_cast<float4 *>(s_in)[q] = __ldcs(reinterpret_cast<const float4 *>(src) + q);
    for (int f = (n4 << 2) + tid; f < nf; f += kMergeBlock) s_in[f] = __ldcs(src + f);
  }
  __syncthreads();
  // keep flags and their ranks inside the tile, in row order (row = k * 256 + tid: k-major, then warp, then lane)
  const float R = a.radius;
  unsigned int ball[kMergeItems];
#pragma unroll
  for (int k = 0; k < kMergeItems; ++k) {
    const int r = k * kMergeBlock + tid;
    bool keep = r < nr;
    if (keep && e > 0) {
      const float x = s_in[r * RD + s_col[0]], y = s_in[r * RD + s_col[1]];
      keep = !(fabsf(x) < R && fabsf(y) < R);  // reader.py:143-150, NaN rows are kept as numpy keeps them
    }
    if (kFrustum && keep) {
      // points_in_convex_polygon_3d_jit: fp32 x, y, z widened to fp64, ((x a + y b) + z c) + d per plane, no FMA
      // contraction; a row is dropped when any plane gives >= 0, so NaN rows are kept and rows on a plane dropped
      const double x = s_in[r * RD + s_col[0]], y = s_in[r * RD + s_col[1]], z = s_in[r * RD + s_col[2]];
#pragma unroll
      for (int p = 0; p < 6; ++p) {
        const double *q = s_pl + 4 * p;
        const double v = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, q[0]), __dmul_rn(y, q[1])), __dmul_rn(z, q[2])), q[3]);
        keep = keep && !(v >= 0.0);
      }
    }
    ball[k] = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_cnt[k * kMergeWarps + wid] = __popc(ball[k]);
  }
  __syncthreads();
  if (wid == 0) {
    const int v = s_cnt[lane];
    int inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += t;
    }
    s_cnt[lane] = inc - v;
    const int aggregate = __shfl_sync(0xffffffffu, inc, 31);
    const int prefix = lookback_exclusive_prefix(scan + 1, s_bid, aggregate);
    if (lane == 0) {
      s_prefix = prefix;
      s_agg = aggregate;
      if (s_bid == gridDim.x - 1) {
        const long long total = static_cast<long long>(prefix) + aggregate;
        n_out[0] = static_cast<int32_t>(total < cap ? total : cap);
        if (total > cap) atomicOr(flags, 1);
      }
    }
  }
  __syncthreads();
  // build the kept rows in shared memory at their rank
  const unsigned int lt = (1u << lane) - 1u;
#pragma unroll
  for (int k = 0; k < kMergeItems; ++k) {
    if (!((ball[k] >> lane) & 1u)) continue;
    const int r = k * kMergeBlock + tid;
    const int o = s_cnt[k * kMergeWarps + wid] + __popc(ball[k] & lt);
    const float *in = s_in + r * RD;
    float *dst = s_out + o * F;
    for (int c = 0; c < a.ncol; ++c) dst[c] = in[s_col[c]];
    if (s_tf) {
      // reader.py:153-157: m.dot(vstack(pts, ones)) in float64, stored back into the fp32 array
      const double x = dst[0], y = dst[1], z = dst[2];
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        double acc = s_m[i * 4 + 0] * x;
        acc = fma(s_m[i * 4 + 1], y, acc);
        acc = fma(s_m[i * 4 + 2], z, acc);
        dst[i] = __double2float_rn(acc + s_m[i * 4 + 3]);
      }
    }
    if (a.use_time_lag) dst[a.ncol] = s_lag;
  }
  __syncthreads();
  // stream the tile's rows [prefix, min(prefix + agg, cap)) out: 16-byte stores between a scalar head and tail
  const long long p0 = s_prefix, p1 = min(static_cast<long long>(s_prefix) + s_agg, cap);
  if (p0 >= p1) return;
  const long long g0 = p0 * F, g1 = p1 * F;
  float *o = out;
  const long long a0 = min((g0 + 3) & ~3ll, g1), a1 = max(a0, g1 & ~3ll);
  for (long long g = g0 + tid; g < a0; g += kMergeBlock) o[g] = s_out[g - g0];
  for (long long q = (a0 >> 2) + tid; q < (a1 >> 2); q += kMergeBlock) {
    const float *s = s_out + (q * 4 - g0);
    __stcs(reinterpret_cast<float4 *>(o) + q, make_float4(s[0], s[1], s[2], s[3]));
  }
  for (long long g = a1 + tid; g < g1; g += kMergeBlock) o[g] = s_out[g - g0];
}

__global__ void __launch_bounds__(256) merge_tail_kernel(float *__restrict__ out, long long cap, int F,
                                                         const int32_t *__restrict__ n_out,
                                                         const int32_t *__restrict__ flags,
                                                         int32_t *__restrict__ status) {
  pdl_trigger();
  pdl_wait();
  const long long g0 = static_cast<long long>(n_out[0]) * F, g1 = cap * F;
  const long long a0 = min((g0 + 3) & ~3ll, g1), a1 = max(a0, g1 & ~3ll);
  const long long tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  if (tid == 0) status[0] = flags[0];
  const float qnan = __int_as_float(0x7fc00000);
  for (long long g = g0 + tid; g < a0; g += stride) out[g] = qnan;
  const float4 n4 = make_float4(qnan, qnan, qnan, qnan);
  for (long long q = (a0 >> 2) + tid; q < (a1 >> 2); q += stride) __stcs(reinterpret_cast<float4 *>(out) + q, n4);
  for (long long g = a1 + tid; g < g1; g += stride) out[g] = qnan;
}

long long merge_tiles(int num_entries, int64_t slot_cap) {
  const long long per = slot_cap > 0 ? (slot_cap + kMergeTile - 1) / kMergeTile : 1;
  return static_cast<long long>(num_entries) * per;
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" size_t p3d_merge_sweeps_workspace_bytes(int num_entries, int64_t slot_cap) {
  if (num_entries < 1 || slot_cap < 0 || merge_tiles(num_entries, slot_cap) >= (1ll << 31)) return 0;
  return carve_merge(nullptr, merge_tiles(num_entries, slot_cap)).bytes;
}

namespace {

template <bool kFrustum>
int merge_sweeps_impl(const float *raw, int num_slots, int64_t slot_cap, int raw_dim, const p3d_sweep_desc *desc,
                      int num_entries, const int32_t *use_dim_host, int n_use_dim, int use_time_lag,
                      float sweep_remove_radius, float *out, int64_t cap, int32_t *n_out_dev, int32_t *status_dev,
                      void *workspace, size_t workspace_bytes, p3d_stream_t stream, const double *planes_dev) {
  if (!desc || !out || !n_out_dev || !status_dev || !workspace || num_entries < 1 || num_slots < 1 || slot_cap < 0 ||
      raw_dim < 3 || n_use_dim < 0 || cap < 0 || (n_use_dim && !use_dim_host) || (!raw && slot_cap))
    return P3D_ERR_INVALID_ARG;
  if ((slot_cap & 3) || (reinterpret_cast<uintptr_t>(raw) & 15) || (reinterpret_cast<uintptr_t>(out) & 15) ||
      (reinterpret_cast<uintptr_t>(workspace) & 255))
    return P3D_ERR_INVALID_ARG;
  if (kFrustum && (!planes_dev || (reinterpret_cast<uintptr_t>(planes_dev) & 7))) return P3D_ERR_INVALID_ARG;
  if (kFrustum && num_entries != 1) return P3D_ERR_UNSUPPORTED;  // the cull is defined on one untransformed cloud
  MergeAttrs a;
  a.raw_dim = raw_dim;
  a.ncol = n_use_dim ? n_use_dim : raw_dim;
  a.use_time_lag = use_time_lag ? 1 : 0;
  a.F = a.ncol + a.use_time_lag;
  a.radius = sweep_remove_radius;
  if (a.ncol < 3) return P3D_ERR_INVALID_ARG;  // the transform and the removal square read columns 0..2
  if (raw_dim + a.F > kMaxCols) return P3D_ERR_UNSUPPORTED;
  for (int c = 0; c < a.ncol; ++c) {
    a.col[c] = n_use_dim ? use_dim_host[c] : c;
    if (a.col[c] < 0 || a.col[c] >= raw_dim) return P3D_ERR_INVALID_ARG;
  }
  for (int c = a.ncol; c < kMaxCols; ++c) a.col[c] = 0;
  if (cap * a.F >= (1ll << 40) || static_cast<double>(num_slots) * slot_cap * raw_dim >= 9.0e15) return P3D_ERR_UNSUPPORTED;
  if (cap >= (1ll << 31)) return P3D_ERR_UNSUPPORTED;  // n_out is an int32
  const long long tiles = merge_tiles(num_entries, slot_cap);
  if (tiles >= (1ll << 31)) return P3D_ERR_UNSUPPORTED;
  const MergeWs w = carve_merge(workspace, tiles);
  if (workspace_bytes < w.bytes) return P3D_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int tpe = static_cast<int>(tiles / num_entries);
  P3D_CUDA_CHECK(cudaMemsetAsync(workspace, 0, w.bytes, st));
  const size_t smem = static_cast<size_t>(kMergeTile) * (raw_dim + a.F) * sizeof(float);
  P3D_CUDA_CHECK(launch_pdl(merge_sweeps_kernel<kFrustum>, dim3(static_cast<unsigned int>(tiles)), dim3(kMergeBlock), smem,
                            st, raw, num_slots, static_cast<long long>(slot_cap), desc, tpe, a, out,
                            static_cast<long long>(cap), w.scan, w.flags, n_out_dev, planes_dev));
  const long long tail = (cap * a.F + 4 * 256 - 1) / (4 * 256);
  const unsigned int tail_blocks = static_cast<unsigned int>(tail < 1 ? 1 : (tail > num_sms() * 4 ? num_sms() * 4 : tail));
  P3D_CUDA_CHECK(launch_pdl(merge_tail_kernel, dim3(tail_blocks), dim3(256), 0, st, out, static_cast<long long>(cap), a.F,
                            static_cast<const int32_t *>(n_out_dev), static_cast<const int32_t *>(w.flags), status_dev));
  return P3D_OK;
}

}  // namespace

extern "C" int p3d_merge_sweeps(const float *raw, int num_slots, int64_t slot_cap, int raw_dim,
                                const p3d_sweep_desc *desc, int num_entries, const int32_t *use_dim_host, int n_use_dim,
                                int use_time_lag, float sweep_remove_radius, float *out, int64_t cap, int32_t *n_out_dev,
                                int32_t *status_dev, void *workspace, size_t workspace_bytes, p3d_stream_t stream) {
  return merge_sweeps_impl<false>(raw, num_slots, slot_cap, raw_dim, desc, num_entries, use_dim_host, n_use_dim,
                                  use_time_lag, sweep_remove_radius, out, cap, n_out_dev, status_dev, workspace,
                                  workspace_bytes, stream, nullptr);
}

extern "C" int p3d_merge_sweeps_frustum(const float *raw, int num_slots, int64_t slot_cap, int raw_dim,
                                        const p3d_sweep_desc *desc, int num_entries, const int32_t *use_dim_host,
                                        int n_use_dim, int use_time_lag, float sweep_remove_radius, float *out,
                                        int64_t cap, int32_t *n_out_dev, int32_t *status_dev, void *workspace,
                                        size_t workspace_bytes, p3d_stream_t stream, const double *planes_dev) {
  return merge_sweeps_impl<true>(raw, num_slots, slot_cap, raw_dim, desc, num_entries, use_dim_host, n_use_dim,
                                 use_time_lag, sweep_remove_radius, out, cap, n_out_dev, status_dev, workspace,
                                 workspace_bytes, stream, planes_dev);
}
