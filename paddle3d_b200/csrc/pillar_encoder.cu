// PillarFeatureNet with one PFNLayer (models/voxel_encoders/pillar_encoder.py:156-210, :81-106; SURVEY.md §8f-2):
// decorate the <= M points of a pillar (xyz - pillar mean, xy - pillar centre), zero the padding rows, Linear(F+5 -> C,
// no bias) + BatchNorm1D(eval) + ReLU, max over the M rows — one block per pillar, one thread per output channel, the
// decorated rows staged in shared memory.  The reference runs this as ~15 elementwise / matmul / argmax launches over
// the [N, M, F+5] and [N, M, C] intermediates; here only voxels [N, M, F] is read and [N, C] written.
// Checked by tests/test_gpu_voxelize.py::test_pillar_feature_net (1e-4 vs the oracle restatement).
#include "common.cuh"
#include "p3d_b200.h"

namespace p3d {
namespace {

constexpr int kMaxM = 64, kMaxF = 8;

__global__ void pfn_kernel(const float *__restrict__ voxels, const int32_t *__restrict__ npv,
                           const int32_t *__restrict__ coors, const int32_t *__restrict__ num_dev, int n_cap, int M, int F,
                           int C, const float *__restrict__ weight, const float *__restrict__ scale,
                           const float *__restrict__ shift, float vx, float vy, float x_off, float y_off,
                           float *__restrict__ out) {
  __shared__ float s_f[kMaxM][kMaxF + 5];
  __shared__ float s_mean[3];
  const int n = num_dev ? min(num_dev[0], n_cap) : n_cap;
  const int i = blockIdx.x;
  if (i >= n) return;
  const int cnt = npv[i];
  const int D = F + 5;
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
    else
      val = v[m * F + (d - F - 3)] - (d == F + 3 ? cx : cy);
    s_f[m][d] = (m < cnt) ? val : 0.f;  // padding rows zeroed after the decoration (:193-198)
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float w[kMaxF + 5];
    for (int d = 0; d < D; ++d) w[d] = __ldg(weight + d * C + c);
    const float sc = __ldg(scale + c), sh = __ldg(shift + c);
    float best = -INFINITY;
    for (int m = 0; m < M; ++m) {
      float acc = 0.f;
      for (int d = 0; d < D; ++d) acc = fmaf(s_f[m][d], w[d], acc);
      best = fmaxf(best, fmaxf(fmaf(acc, sc, sh), 0.f));
    }
    out[static_cast<size_t>(i) * C + c] = best;
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
  pfn_kernel<<<static_cast<unsigned int>(n_cap), threads, 0, static_cast<cudaStream_t>(stream)>>>(
      voxels, num_points_per_voxel, coors, num_voxels_dev, static_cast<int>(n_cap), max_points, num_point_dim,
      out_channels, weight, bn_scale, bn_shift, vx, vy, x_off, y_off, out);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
