// Dense BEV canvas writer for sm_90a: PointPillarsScatter and sparse to_dense(+transpose), gather-formulated.
//
// The reference does zeros + paddle.scatter + transpose (pillar_scatter.py:71-92) or
// to_dense + transpose + reshape (sparse_resnet.py:202-206): three passes over the dense tensor.
// Here the dense output [batch, C, D, ny, nx] is written exactly once:
//   S1 memset      cell -> row map <- -1                                  (4 B per cell)
//   S2 scat_map    map[cell(row)] = max(row)   (later rows win on duplicates, as scatter-overwrite)
//   S3 scat_write  one CTA per tile of 128 consecutive cells: every channel row of the tile is written with one
//                  float4 per lane (512 B per warp store); an occupied cell's value is gathered from its feature
//                  row (8 consecutive channels per warp: L1 sector reuse), empty cells are just the store.
// Algorithmic bytes: 4*n*C (features) + 16*n (coords) + 4*batch*C*D*ny*nx (canvas).
#include "common.cuh"

namespace p3d {
namespace {

constexpr int kTile = 128;         // cells per CTA

__global__ void __launch_bounds__(256) scat_map_kernel(const int32_t *__restrict__ coords,
                                                       const int32_t *__restrict__ n_dev, int n_cap, int batch, int D,
                                                       int ny, int nx, int use_z, int32_t *__restrict__ map) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = n_dev ? min(n_dev[0], n_cap) : n_cap;
  if (i >= n) return;
  const int4 c = *reinterpret_cast<const int4 *>(coords + static_cast<size_t>(i) * 4);
  const int z = use_z ? c.y : 0;
  if (c.x < 0 || c.x >= batch || z < 0 || z >= D || c.z < 0 || c.z >= ny || c.w < 0 || c.w >= nx) return;
  atomicMax(&map[((static_cast<size_t>(c.x) * D + z) * ny + c.z) * nx + c.w], i);
}

// One CTA per tile of 128 consecutive cells.  The tile's 128 map entries are read once; then every warp emits whole
// channel rows of the tile (512 bytes per warp store, streaming): a lane holds 4 consecutive cells and fetches the
// value of an occupied cell straight from the feature row (`feats[row * C + c]`: warp w walks 8 CONSECUTIVE channels, so
// the 4-byte gathers of a cell hit the 32-byte sector its first channel brought into L1).  Empty cells (94 % of a
// PointPillars canvas) cost nothing but the store.  Round 1 staged the occupied rows channel-major in 33 KB of shared
// memory first: two block barriers and a dependent load on the critical path of every tile, 6 CTAs per SM; without the
// staging the stores of the empty cells are issued as soon as the map entries arrive and 8 CTAs fit.
template <bool kVec>
__global__ void __launch_bounds__(256) scat_write_kernel(const float *__restrict__ feats,
                                                         const int32_t *__restrict__ map, int C, long long S,
                                                         float *__restrict__ out) {
  __shared__ int s_row[kTile];
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.y;
  const long long cell0 = static_cast<long long>(blockIdx.x) * kTile;
  const int ncell = static_cast<int>(min(static_cast<long long>(kTile), S - cell0));
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid < kTile) s_row[tid] = tid < ncell ? __ldg(map + static_cast<size_t>(b) * S + cell0 + tid) : -1;
  __syncthreads();
  if (kVec) {
    const int k = lane * 4;
    if (k >= ncell) return;  // S % 4 == 0 => ncell % 4 == 0
    const int r0 = s_row[k], r1 = s_row[k + 1], r2 = s_row[k + 2], r3 = s_row[k + 3];
    const bool any = (r0 & r1 & r2 & r3) >= 0;  // some row index non-negative
    // channels in blocks of 8 consecutive ones per warp: c = 64 i + 8 wid + j
    for (int cb = wid * 8; cb < C; cb += 64) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = cb + j;
        if (c >= C) break;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (any) {
          if (r0 >= 0) v.x = __ldg(feats + static_cast<size_t>(r0) * C + c);
          if (r1 >= 0) v.y = __ldg(feats + static_cast<size_t>(r1) * C + c);
          if (r2 >= 0) v.z = __ldg(feats + static_cast<size_t>(r2) * C + c);
          if (r3 >= 0) v.w = __ldg(feats + static_cast<size_t>(r3) * C + c);
        }
        __stcs(reinterpret_cast<float4 *>(out + (static_cast<size_t>(b) * C + c) * S + cell0 + k), v);
      }
    }
  } else {
    for (int c = wid; c < C; c += 8) {
      float *dst = out + (static_cast<size_t>(b) * C + c) * S + cell0;
      for (int k = lane; k < ncell; k += 32) {
        const int r = s_row[k];
        dst[k] = r >= 0 ? __ldg(feats + static_cast<size_t>(r) * C + c) : 0.f;
      }
    }
  }
}

// Sparse rows (fp16-pair H16 rows of C channels, C % 32 == 0) -> pixel H16 image [batch, ny, nx][D * C channels]: the
// fp16-pair form of SparseResNet3D's to_dense + transpose + reshape (sparse_resnet.py:202-206, channel = z * C + c) that
// the dense RPN consumes directly (no fp32 NCHW tensor, no layout conversion pass).  One warp copies one row (4 * C bytes).
__global__ void __launch_bounds__(256) rows_to_pixel_h16_kernel(const uint4 *__restrict__ rows, const int32_t *__restrict__ coords,
                                                                const int32_t *__restrict__ n_dev, int n_cap, int C, int batch,
                                                                int D, int ny, int nx, uint4 *__restrict__ out) {
  const int n = n_dev ? min(n_dev[0], n_cap) : n_cap;
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= n) return;
  const int4 c = *reinterpret_cast<const int4 *>(coords + static_cast<size_t>(r) * 4);
  if (c.x < 0 || c.x >= batch || c.y < 0 || c.y >= D || c.z < 0 || c.z >= ny || c.w < 0 || c.w >= nx) return;
  const int q_row = C / 4;  // uint4 per row (4 * C bytes)
  uint4 *dst = out + ((static_cast<size_t>(c.x) * ny + c.z) * nx + c.w) * (static_cast<size_t>(D) * q_row) + static_cast<size_t>(c.y) * q_row;
  const uint4 *src = rows + static_cast<size_t>(r) * q_row;
  for (int q = lane; q < q_row; q += 32) dst[q] = __ldg(src + q);
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_sparse_rows_to_pixel_h16(const void *rows_h16, const int32_t *coords, const int32_t *n_dev, int n_cap, int C,
                                            int batch, int D, int ny, int nx, void *out_pixel_h16, p3d_stream_t stream) {
  if (n_cap < 0 || C < 32 || C % 32 || batch < 1 || D < 1 || ny < 1 || nx < 1 || !out_pixel_h16 || (n_cap && (!rows_h16 || !coords)))
    return P3D_ERR_INVALID_ARG;
  if ((reinterpret_cast<uintptr_t>(rows_h16) & 15) || (reinterpret_cast<uintptr_t>(coords) & 15) ||
      (reinterpret_cast<uintptr_t>(out_pixel_h16) & 15))
    return P3D_ERR_INVALID_ARG;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t bytes = static_cast<size_t>(batch) * ny * nx * D * C * 4;
  P3D_CUDA_CHECK(cudaMemsetAsync(out_pixel_h16, 0, bytes, st));  // (hi, lo') = (0, 0) is the value 0
  if (n_cap > 0) {
    rows_to_pixel_h16_kernel<<<div_up(static_cast<long long>(n_cap) * 32, 256), 256, 0, st>>>(
        static_cast<const uint4 *>(rows_h16), coords, n_dev, n_cap, C, batch, D, ny, nx, static_cast<uint4 *>(out_pixel_h16));
    P3D_LAUNCH_CHECK();
  }
  return P3D_OK;
}

extern "C" size_t p3d_scatter_dense_workspace_bytes(int batch, int D, int ny, int nx) {
  if (batch < 1 || D < 1 || ny < 1 || nx < 1) return 0;
  return align_up(static_cast<size_t>(batch) * D * ny * nx * sizeof(int32_t));
}

extern "C" int p3d_scatter_dense(const float *feats, const int32_t *coords, const int32_t *n_dev, int n_cap, int C,
                                 int batch, int D, int ny, int nx, int use_z, float *out, void *workspace,
                                 size_t workspace_bytes, p3d_stream_t stream) {
  if (n_cap < 0 || C < 1 || batch < 1 || D < 1 || ny < 1 || nx < 1 || !out || !workspace ||
      (n_cap && (!feats || !coords)))
    return P3D_ERR_INVALID_ARG;
  if (batch > 65535) return P3D_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(coords) & 15) || (reinterpret_cast<uintptr_t>(out) & 15)) return P3D_ERR_INVALID_ARG;
  const size_t need = p3d_scatter_dense_workspace_bytes(batch, D, ny, nx);
  if (workspace_bytes < need) return P3D_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int32_t *map = static_cast<int32_t *>(workspace);
  const long long S = static_cast<long long>(D) * ny * nx;
  P3D_CUDA_CHECK(cudaMemsetAsync(map, 0xff, static_cast<size_t>(batch) * S * sizeof(int32_t), st));
  if (n_cap > 0) {
    scat_map_kernel<<<div_up(n_cap, 256), 256, 0, st>>>(coords, n_dev, n_cap, batch, D, ny, nx, use_z, map);
    P3D_LAUNCH_CHECK();
  }
  dim3 grid(div_up(S, kTile), batch);
  if (S % 4 == 0)
    P3D_CUDA_CHECK(launch_pdl(scat_write_kernel<true>, grid, dim3(256), 0, st, feats, static_cast<const int32_t *>(map), C, S, out));
  else
    P3D_CUDA_CHECK(launch_pdl(scat_write_kernel<false>, grid, dim3(256), 0, st, feats, static_cast<const int32_t *>(map), C, S, out));
  return P3D_OK;
}
