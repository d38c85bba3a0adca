// PillarFeatureNet with one or two PFNLayers (models/voxel_encoders/pillar_encoder.py:156-210, :81-106; SURVEY.md §8f-2):
// decorate the <= M points of a pillar (xyz - pillar mean, xy - pillar centre), zero the padding rows, then
//   one layer  (last):          Linear(F+5 -> C, no bias) + BatchNorm1D(eval) + ReLU, max over the M rows;
//   two layers (first, last):   Linear(F+5 -> C1) + BN + ReLU -> x [M, C1], x_max = max over the rows, per row
//                               concat([x, x_max]) -> Linear(2 C1 -> C2) + BN + ReLU, max over the rows.
// One block per pillar, the decorated rows (and the first layer's rows) staged in shared memory.  The reference runs this
// as ~15 elementwise / matmul / argmax launches over the [N, M, F+5] and [N, M, C] intermediates; here only voxels
// [N, M, F] is read and [N, C] written.  Checked by tests/test_gpu_lidar_front_end.py::test_pillar_feature_net_one_layer
// (one layer: F 3 .. 8, M 1 .. 64, C 1 .. 200, far pillars, padding rows deciding the max, rows beyond the count
// untouched), tests/test_gpu_voxelize.py::test_pillar_feature_net and tests/test_gpu_centerpoint_pillars.py (two layers),
// tests/test_gpu_bevfusion.py::test_hard_vfe_matches_fp64 (HardVFE),
// 1e-4 vs the oracle restatements; the argument limits by tests/test_lidar_front_end_oracle.py.  The wide two-layer
// instantiation (kMaxRows = 128, p3d_pillar_feature_net2_wide, CenterPoint-pillars KITTI's 100 points per pillar) by
// tests/test_gpu_centerpoint_pillars_kitti.py, its limits by tests/test_centerpoint_pillars_kitti.py.
#include "common.cuh"
#include "p3d_b200.h"

namespace p3d {
namespace {

constexpr int kMaxM = 64, kMaxMWide = 128, kMaxF = 8, kMaxMid = 64;

// kLayers = 1: C1 = C is the output width and (C2, w2, scale2, shift2) are unused.  kLayers = 2: C1 is the first
// layer's width (<= kMaxMid), w2 is [2 C1, C2].  kVoxelZ (HardVFE, with kLayers = 2): the decoration also carries
// z - (coors_z * vz + z_off), so a row has F + 6 features.  kMaxRows: the most points per pillar the shared-memory
// staging holds (M <= kMaxRows); it sizes the arrays only, the arithmetic and its order do not depend on it.
template <int kLayers, bool kVoxelZ = false, int kMaxRows = kMaxM>
__global__ void pfn_kernel(const float *__restrict__ voxels, const int32_t *__restrict__ npv,
                           const int32_t *__restrict__ coors, const int32_t *__restrict__ num_dev, int n_cap, int M, int F,
                           int C1, const float *__restrict__ weight, const float *__restrict__ scale,
                           const float *__restrict__ shift, int C2, const float *__restrict__ w2,
                           const float *__restrict__ scale2, const float *__restrict__ shift2, float vx, float vy,
                           float x_off, float y_off, float *__restrict__ out, float vz = 0.f, float z_off = 0.f) {
  constexpr int kExtra = kVoxelZ ? 6 : 5;
  __shared__ float s_f[kMaxRows][kMaxF + kExtra];
  __shared__ float s_mean[3];
  const int n = num_dev ? min(num_dev[0], n_cap) : n_cap;
  const int i = blockIdx.x;
  if (i >= n) return;
  const int cnt = npv[i];
  const int D = F + kExtra;
  const float *v = voxels + static_cast<size_t>(i) * M * F;
  if (threadIdx.x < 3) {  // mean over ALL M rows' sum (padding rows are zero) divided by the point count (:172-175)
    float s = 0.f;
    for (int m = 0; m < M; ++m) s += v[m * F + threadIdx.x];
    s_mean[threadIdx.x] = s / static_cast<float>(cnt);
  }
  __syncthreads();
  const float cx = static_cast<float>(coors[i * 4 + 3]) * vx + x_off, cy = static_cast<float>(coors[i * 4 + 2]) * vy + y_off;
  for (int e = threadIdx.x; e < M * D; e += blockDim.x) {
    const int m = e / D, d = e - m * D;
    float val;
    if (d < F)
      val = v[m * F + d];
    else if (d < F + 3)
      val = v[m * F + (d - F)] - s_mean[d - F];
    else if constexpr (kVoxelZ)
      val = v[m * F + (d - F - 3)] -
            (d == F + 3 ? cx : d == F + 4 ? cy : static_cast<float>(coors[i * 4 + 1]) * vz + z_off);
    else
      val = v[m * F + (d - F - 3)] - (d == F + 3 ? cx : cy);
    s_f[m][d] = (m < cnt) ? val : 0.f;  // padding rows zeroed after the decoration (:193-198)
  }
  __syncthreads();
  if constexpr (kLayers == 1) {
    for (int c = threadIdx.x; c < C1; c += blockDim.x) {
      float w[kMaxF + 5];
      for (int d = 0; d < D; ++d) w[d] = __ldg(weight + d * C1 + c);
      const float sc = __ldg(scale + c), sh = __ldg(shift + c);
      float best = -INFINITY;
      for (int m = 0; m < M; ++m) {
        float acc = 0.f;
        for (int d = 0; d < D; ++d) acc = fmaf(s_f[m][d], w[d], acc);
        best = fmaxf(best, fmaxf(fmaf(acc, sc, sh), 0.f));
      }
      out[static_cast<size_t>(i) * C1 + c] = best;
    }
  } else {
    __shared__ float s_x[kMaxRows][kMaxMid];
    __shared__ float s_xmax[kMaxMid];
    // Every padding row has the same (zero) decorated input, so the first padding row (row cnt, when cnt < M) stands
    // for all of them: in layer 1 its value ReLU(shift1) enters x_max, in layer 2 its output enters the final max.
    const int rows = min(cnt + 1, M);
    for (int e = threadIdx.x; e < rows * C1; e += blockDim.x) {
      const int m = e / C1, c = e - m * C1;
      float acc = 0.f;
      for (int d = 0; d < D; ++d) acc = fmaf(s_f[m][d], __ldg(weight + d * C1 + c), acc);
      s_x[m][c] = fmaxf(fmaf(acc, __ldg(scale + c), __ldg(shift + c)), 0.f);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C1; c += blockDim.x) {
      float best = -INFINITY;
      for (int m = 0; m < rows; ++m) best = fmaxf(best, s_x[m][c]);
      s_xmax[c] = best;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C2; c += blockDim.x) {
      // W2 rows C1..2 C1 multiply x_max, the same for every row of the pillar: that half of the product once per pillar
      float base = 0.f;
      for (int k = 0; k < C1; ++k) base = fmaf(s_xmax[k], __ldg(w2 + (C1 + k) * C2 + c), base);
      float w[kMaxMid];
#pragma unroll
      for (int k = 0; k < kMaxMid; ++k) w[k] = k < C1 ? __ldg(w2 + k * C2 + c) : 0.f;
      const float sc = __ldg(scale2 + c), sh = __ldg(shift2 + c);
      float best = -INFINITY;
      for (int m = 0; m < rows; ++m) {
        float acc = base;
#pragma unroll
        for (int k = 0; k < kMaxMid; ++k)
          if (k < C1) acc = fmaf(s_x[m][k], w[k], acc);
        best = fmaxf(best, fmaxf(fmaf(acc, sc, sh), 0.f));
      }
      out[static_cast<size_t>(i) * C2 + c] = best;
    }
  }
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_pillar_feature_net(const float *voxels, const int32_t *num_points_per_voxel, const int32_t *coors,
                                      const int32_t *num_voxels_dev, int64_t n_cap, int max_points, int num_point_dim,
                                      int out_channels, const float *weight, const float *bn_scale,
                                      const float *bn_shift, const float *voxel_size_host,
                                      const float *point_cloud_range_host, float *out, p3d_stream_t stream) {
  if (!voxels || !num_points_per_voxel || !coors || !weight || !bn_scale || !bn_shift || !voxel_size_host ||
      !point_cloud_range_host || !out || n_cap < 0 || out_channels < 1)
    return P3D_ERR_INVALID_ARG;
  if (max_points < 1 || max_points > kMaxM || num_point_dim < 3 || num_point_dim > kMaxF) return P3D_ERR_UNSUPPORTED;
  if (n_cap == 0) return P3D_OK;
  const float vx = voxel_size_host[0], vy = voxel_size_host[1];
  const float x_off = vx / 2 + point_cloud_range_host[0], y_off = vy / 2 + point_cloud_range_host[1];  // :147-148
  const int threads = out_channels <= 64 ? 64 : 128;
  pfn_kernel<1><<<static_cast<unsigned int>(n_cap), threads, 0, static_cast<cudaStream_t>(stream)>>>(
      voxels, num_points_per_voxel, coors, num_voxels_dev, static_cast<int>(n_cap), max_points, num_point_dim,
      out_channels, weight, bn_scale, bn_shift, 0, nullptr, nullptr, nullptr, vx, vy, x_off, y_off, out);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

namespace {

template <int kMaxRows>
int launch_pfn2(const float *voxels, const int32_t *num_points_per_voxel, const int32_t *coors,
                const int32_t *num_voxels_dev, int64_t n_cap, int max_points, int num_point_dim, int mid_channels,
                const float *weight1, const float *bn_scale1, const float *bn_shift1, int out_channels,
                const float *weight2, const float *bn_scale2, const float *bn_shift2, const float *voxel_size_host,
                const float *point_cloud_range_host, float *out, p3d_stream_t stream) {
  if (!voxels || !num_points_per_voxel || !coors || !weight1 || !bn_scale1 || !bn_shift1 || !weight2 || !bn_scale2 ||
      !bn_shift2 || !voxel_size_host || !point_cloud_range_host || !out || n_cap < 0 || mid_channels < 1 ||
      out_channels < 1)
    return P3D_ERR_INVALID_ARG;
  if (max_points < 1 || max_points > kMaxRows || num_point_dim < 3 || num_point_dim > kMaxF || mid_channels > kMaxMid)
    return P3D_ERR_UNSUPPORTED;
  if (n_cap == 0) return P3D_OK;
  const float vx = voxel_size_host[0], vy = voxel_size_host[1];
  const float x_off = vx / 2 + point_cloud_range_host[0], y_off = vy / 2 + point_cloud_range_host[1];
  const int threads = out_channels <= 64 ? 64 : 128;
  pfn_kernel<2, false, kMaxRows><<<static_cast<unsigned int>(n_cap), threads, 0, static_cast<cudaStream_t>(stream)>>>(
      voxels, num_points_per_voxel, coors, num_voxels_dev, static_cast<int>(n_cap), max_points, num_point_dim,
      mid_channels, weight1, bn_scale1, bn_shift1, out_channels, weight2, bn_scale2, bn_shift2, vx, vy, x_off, y_off,
      out);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

}  // namespace

extern "C" int p3d_pillar_feature_net2(const float *voxels, const int32_t *num_points_per_voxel, const int32_t *coors,
                                       const int32_t *num_voxels_dev, int64_t n_cap, int max_points, int num_point_dim,
                                       int mid_channels, const float *weight1, const float *bn_scale1,
                                       const float *bn_shift1, int out_channels, const float *weight2,
                                       const float *bn_scale2, const float *bn_shift2, const float *voxel_size_host,
                                       const float *point_cloud_range_host, float *out, p3d_stream_t stream) {
  return launch_pfn2<kMaxM>(voxels, num_points_per_voxel, coors, num_voxels_dev, n_cap, max_points, num_point_dim,
                            mid_channels, weight1, bn_scale1, bn_shift1, out_channels, weight2, bn_scale2, bn_shift2,
                            voxel_size_host, point_cloud_range_host, out, stream);
}

extern "C" int p3d_pillar_feature_net2_wide(const float *voxels, const int32_t *num_points_per_voxel,
                                            const int32_t *coors, const int32_t *num_voxels_dev, int64_t n_cap,
                                            int max_points, int num_point_dim, int mid_channels, const float *weight1,
                                            const float *bn_scale1, const float *bn_shift1, int out_channels,
                                            const float *weight2, const float *bn_scale2, const float *bn_shift2,
                                            const float *voxel_size_host, const float *point_cloud_range_host,
                                            float *out, p3d_stream_t stream) {
  return launch_pfn2<kMaxMWide>(voxels, num_points_per_voxel, coors, num_voxels_dev, n_cap, max_points, num_point_dim,
                                mid_channels, weight1, bn_scale1, bn_shift1, out_channels, weight2, bn_scale2,
                                bn_shift2, voxel_size_host, point_cloud_range_host, out, stream);
}

extern "C" int p3d_hard_vfe(const float *voxels, const int32_t *num_points_per_voxel, const int32_t *coors,
                            const int32_t *num_voxels_dev, int64_t n_cap, int max_points, int num_point_dim,
                            int mid_channels, const float *weight1, const float *bn_scale1, const float *bn_shift1,
                            int out_channels, const float *weight2, const float *bn_scale2, const float *bn_shift2,
                            const float *voxel_size_host, const float *point_cloud_range_host, float *out,
                            p3d_stream_t stream) {
  if (!voxels || !num_points_per_voxel || !coors || !weight1 || !bn_scale1 || !bn_shift1 || !weight2 || !bn_scale2 ||
      !bn_shift2 || !voxel_size_host || !point_cloud_range_host || !out || n_cap < 0 || mid_channels < 1 ||
      out_channels < 1)
    return P3D_ERR_INVALID_ARG;
  if (max_points < 1 || max_points > kMaxM || num_point_dim < 3 || num_point_dim > kMaxF || mid_channels > kMaxMid)
    return P3D_ERR_UNSUPPORTED;
  if (n_cap == 0) return P3D_OK;
  const float vx = voxel_size_host[0], vy = voxel_size_host[1], vz = voxel_size_host[2];
  const float x_off = vx / 2 + point_cloud_range_host[0], y_off = vy / 2 + point_cloud_range_host[1];
  const float z_off = vz / 2 + point_cloud_range_host[2];  // HardVFE's voxel centre includes z
  const int threads = out_channels <= 64 ? 64 : 128;
  pfn_kernel<2, true><<<static_cast<unsigned int>(n_cap), threads, 0, static_cast<cudaStream_t>(stream)>>>(
      voxels, num_points_per_voxel, coors, num_voxels_dev, static_cast<int>(n_cap), max_points, num_point_dim,
      mid_channels, weight1, bn_scale1, bn_shift1, out_channels, weight2, bn_scale2, bn_shift2, vx, vy, x_off, y_off,
      out, vz, z_off);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
