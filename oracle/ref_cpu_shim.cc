// TEST INFRASTRUCTURE ONLY — not part of the product.
// extern "C" entry points around the UNMODIFIED reference CPU ops, which are
// compiled from where they lie in a Paddle3D checkout ($P3D_REFERENCE) by oracle/Makefile:
//   paddle3d/ops/voxel/voxelize_op.cc:84-146   hard_voxelize_cpu
//   paddle3d/ops/iou3d_nms/iou3d_cpu.cpp:241-264  boxes_iou_bev_cpu
// The wrappers only marshal raw host pointers into the stub paddle::Tensor.
#include <cstring>
#include <vector>

#include "paddle/extension.h"

std::vector<paddle::Tensor> hard_voxelize_cpu(const paddle::Tensor &points, const std::vector<float> &voxel_size,
                                              const std::vector<float> &point_cloud_range,
                                              const int max_num_points_in_voxel, const int max_voxels);
std::vector<paddle::Tensor> boxes_iou_bev_cpu(const paddle::Tensor &boxes_a_tensor,
                                              const paddle::Tensor &boxes_b_tensor);

extern "C" {

int ref_hard_voxelize_cpu(const float *points, long long num_points, int num_point_dim, const float *voxel_size,
                          const float *pc_range, int max_points, int max_voxels, float *voxels, int *coords,
                          int *num_points_per_voxel, int *num_voxels) {
  paddle::Tensor pts(const_cast<float *>(points), {num_points, num_point_dim}, paddle::DataType::FLOAT32);
  std::vector<float> vs(voxel_size, voxel_size + 3), pcr(pc_range, pc_range + 6);
  auto outs = hard_voxelize_cpu(pts, vs, pcr, max_points, max_voxels);
  std::memcpy(voxels, outs[0].data<float>(), sizeof(float) * outs[0].size());
  std::memcpy(coords, outs[1].data<int>(), sizeof(int) * outs[1].size());
  std::memcpy(num_points_per_voxel, outs[2].data<int>(), sizeof(int) * outs[2].size());
  num_voxels[0] = outs[3].data<int>()[0];
  return 0;
}

int ref_boxes_iou_bev_cpu(const float *boxes_a, int num_a, const float *boxes_b, int num_b, float *iou) {
  paddle::Tensor a(const_cast<float *>(boxes_a), {num_a, 7}, paddle::DataType::FLOAT32);
  paddle::Tensor b(const_cast<float *>(boxes_b), {num_b, 7}, paddle::DataType::FLOAT32);
  auto outs = boxes_iou_bev_cpu(a, b);
  std::memcpy(iou, outs[0].data<float>(), sizeof(float) * (size_t)num_a * num_b);
  return 0;
}
}
