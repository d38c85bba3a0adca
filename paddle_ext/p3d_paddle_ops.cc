// Paddle custom-op glue: the SAME registrations (op names, inputs, outputs, attrs, infer functions) as the
// reference's hot-path ops, with kernel functions that call the C ABI of libp3d_b200.so.
//
//   hard_voxelize            paddle3d/ops/voxel/voxelize_op.cc:183-191
//   boxes_iou_bev_gpu, boxes_overlap_bev_gpu, nms_gpu, nms_normal_gpu
//                            paddle3d/ops/iou3d_nms/iou3d_nms_api.cpp:73-108
//   centerpoint_postprocess  paddle3d/ops/centerpoint_postprocess/postprocess.cc:91-104
//   bev_pool_v2              paddle3d/ops/bev_pool_v2/bev_pool.cc:111-118
//   bev_pool_v2_bkwd         paddle3d/ops/bev_pool_v2_backward/bev_pool_bkwd.cc:75-80
//
// Build (where PaddlePaddle exists): list this file as the `sources` of the op in paddle3d/ops/__init__.py and
// add  extra_ldflags=['-L<repo>/paddle3d_b200', '-lp3d_b200']  — see INTEGRATION.md.  In this repository
// PaddlePaddle is not installable, so the file is compile-checked against oracle/stub/paddle/extension.h
// (tests/test_abi.py::test_paddle_glue_compiles) and the C ABI itself is exercised through ctypes.
#include <vector>

#include "paddle/extension.h"
#include "p3d_b200.h"

#define P3D_CHECK_GPU(x) PD_CHECK((x).is_gpu() || (x).is_gpu_pinned(), #x " must be a GPU Tensor.")
#define P3D_CALL(expr)                                                                 \
  do {                                                                                 \
    int _rc = (expr);                                                                  \
    if (_rc != 0) PD_THROW(std::string(#expr " failed: ") + p3d_status_string(_rc)); \
  } while (0)

namespace {

paddle::Tensor workspace(size_t bytes) {
  return paddle::empty({static_cast<int64_t>(bytes ? bytes : 256)}, paddle::DataType::UINT8, paddle::GPUPlace());
}

}  // namespace

// ---------------------------------------------------------------- hard_voxelize
std::vector<paddle::Tensor> hard_voxelize(const paddle::Tensor &points, const std::vector<float> &voxel_size,
                                          const std::vector<float> &point_cloud_range,
                                          const int max_num_points_in_voxel, const int max_voxels) {
  P3D_CHECK_GPU(points);  // this build has no CPUPlace kernel: the reference's CPU branch (voxelize_op.cc:153-155) throws here
  const int64_t n = points.shape()[0];
  const int f = static_cast<int>(points.shape()[1]);
  auto voxels = paddle::empty({max_voxels, max_num_points_in_voxel, f}, paddle::DataType::FLOAT32, paddle::GPUPlace());
  auto coords = paddle::empty({max_voxels, 3}, paddle::DataType::INT32, paddle::GPUPlace());
  auto npv = paddle::empty({max_voxels}, paddle::DataType::INT32, paddle::GPUPlace());
  auto num_voxels = paddle::empty({1}, paddle::DataType::INT32, paddle::GPUPlace());
  const size_t ws_bytes = p3d_hard_voxelize_workspace_bytes(n, max_num_points_in_voxel, max_voxels);
  auto ws = workspace(ws_bytes);
  P3D_CALL(p3d_hard_voxelize(points.data<float>(), n, f, voxel_size.data(), point_cloud_range.data(),
                             max_num_points_in_voxel, max_voxels, voxels.data<float>(), coords.data<int>(),
                             npv.data<int>(), num_voxels.data<int>(), ws.data<uint8_t>(), ws_bytes, points.stream()));
  return {voxels, coords, npv, num_voxels};
}

std::vector<std::vector<int64_t>> HardInferShape(std::vector<int64_t> points_shape, const std::vector<float> &voxel_size,
                                                 const std::vector<float> &point_cloud_range,
                                                 const int &max_num_points_in_voxel, const int &max_voxels) {
  return {{max_voxels, max_num_points_in_voxel, points_shape[1]}, {max_voxels, 3}, {max_voxels}, {1}};
}

std::vector<paddle::DataType> HardInferDtype(paddle::DataType points_dtype) {
  return {points_dtype, paddle::DataType::INT32, paddle::DataType::INT32, paddle::DataType::INT32};
}

PD_BUILD_OP(hard_voxelize)
    .Inputs({"POINTS"})
    .Outputs({"VOXELS", "COORS", "NUM_POINTS_PER_VOXEL", "num_voxels"})
    .SetKernelFn(PD_KERNEL(hard_voxelize))
    .Attrs({"voxel_size: std::vector<float>", "point_cloud_range: std::vector<float>", "max_num_points_in_voxel: int",
            "max_voxels: int"})
    .SetInferShapeFn(PD_INFER_SHAPE(HardInferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(HardInferDtype));

// ---------------------------------------------------------------- iou3d_nms
static std::vector<paddle::Tensor> pairwise(const paddle::Tensor &a, const paddle::Tensor &b, bool iou) {
  P3D_CHECK_GPU(a);
  P3D_CHECK_GPU(b);
  const int na = static_cast<int>(a.shape()[0]), nb = static_cast<int>(b.shape()[0]);
  auto out = paddle::empty({na, nb}, paddle::DataType::FLOAT32, paddle::GPUPlace());
  if (iou)
    P3D_CALL(p3d_boxes_iou_bev(a.data<float>(), na, b.data<float>(), nb, out.data<float>(), a.stream()));
  else
    P3D_CALL(p3d_boxes_overlap_bev(a.data<float>(), na, b.data<float>(), nb, out.data<float>(), a.stream()));
  return {out};
}
std::vector<paddle::Tensor> boxes_iou_bev_gpu(const paddle::Tensor &a, const paddle::Tensor &b) { return pairwise(a, b, true); }
std::vector<paddle::Tensor> boxes_overlap_bev_gpu(const paddle::Tensor &a, const paddle::Tensor &b) {
  return pairwise(a, b, false);
}

static std::vector<paddle::Tensor> nms_any(const paddle::Tensor &boxes, float thresh, int normal) {
  P3D_CHECK_GPU(boxes);
  const int n = static_cast<int>(boxes.shape()[0]);
  auto keep_dev = paddle::empty({n > 0 ? n : 1}, paddle::DataType::INT32, paddle::GPUPlace());
  auto num_dev = paddle::empty({1}, paddle::DataType::INT32, paddle::GPUPlace());
  const size_t ws_bytes = p3d_nms_workspace_bytes(n);
  auto ws = workspace(ws_bytes);
  P3D_CALL(p3d_nms(boxes.data<float>(), n, thresh, normal, keep_dev.data<int>(), num_dev.data<int>(),
                   ws.data<uint8_t>(), ws_bytes, boxes.stream()));
  // the reference returns CPU tensors (iou3d_nms.cpp:89-92); one blocking copy of the result, none of the matrix
  return {keep_dev.copy_to(paddle::CPUPlace(), true), num_dev.copy_to(paddle::CPUPlace(), true)};
}
std::vector<paddle::Tensor> nms_gpu(const paddle::Tensor &boxes, float nms_overlap_thresh) {
  return nms_any(boxes, nms_overlap_thresh, 0);
}
std::vector<paddle::Tensor> nms_normal_gpu(const paddle::Tensor &boxes, float nms_overlap_thresh) {
  return nms_any(boxes, nms_overlap_thresh, 1);
}

std::vector<paddle::DataType> PairInferDtype(paddle::DataType a, paddle::DataType b) { return {a}; }
std::vector<std::vector<int64_t>> PairInferShape(std::vector<int64_t> a, std::vector<int64_t> b) { return {{a[0], b[0]}}; }
std::vector<paddle::DataType> NmsInferDtype(paddle::DataType boxes_dtype) {
  return {paddle::DataType::INT64, paddle::DataType::INT64};  // as declared by the reference (api.cpp:34-36)
}
std::vector<std::vector<int64_t>> NmsInferShape(std::vector<int64_t> boxes_shape) { return {{boxes_shape[0]}, {1}}; }

PD_BUILD_OP(boxes_iou_bev_gpu)
    .Inputs({"boxes_a_tensor", " boxes_b_tensor"})
    .Outputs({"ans_iou_tensor"})
    .SetKernelFn(PD_KERNEL(boxes_iou_bev_gpu))
    .SetInferDtypeFn(PD_INFER_DTYPE(PairInferDtype))
    .SetInferShapeFn(PD_INFER_SHAPE(PairInferShape));
PD_BUILD_OP(boxes_overlap_bev_gpu)
    .Inputs({"boxes_a", " boxes_b"})
    .Outputs({"ans_overlap"})
    .SetKernelFn(PD_KERNEL(boxes_overlap_bev_gpu))
    .SetInferDtypeFn(PD_INFER_DTYPE(PairInferDtype))
    .SetInferShapeFn(PD_INFER_SHAPE(PairInferShape));
PD_BUILD_OP(nms_gpu)
    .Inputs({"boxes"})
    .Outputs({"keep", "num_to_keep"})
    .Attrs({"nms_overlap_thresh: float"})
    .SetKernelFn(PD_KERNEL(nms_gpu))
    .SetInferDtypeFn(PD_INFER_DTYPE(NmsInferDtype))
    .SetInferShapeFn(PD_INFER_SHAPE(NmsInferShape));
PD_BUILD_OP(nms_normal_gpu)
    .Inputs({"boxes"})
    .Outputs({"keep", "num_to_keep"})
    .Attrs({"nms_overlap_thresh: float"})
    .SetKernelFn(PD_KERNEL(nms_normal_gpu))
    .SetInferDtypeFn(PD_INFER_DTYPE(NmsInferDtype))
    .SetInferShapeFn(PD_INFER_SHAPE(NmsInferShape));

// ---------------------------------------------------------------- centerpoint_postprocess
std::vector<paddle::Tensor> centerpoint_postprocess(
    const std::vector<paddle::Tensor> &hm, const std::vector<paddle::Tensor> &reg,
    const std::vector<paddle::Tensor> &height, const std::vector<paddle::Tensor> &dim,
    const std::vector<paddle::Tensor> &vel, const std::vector<paddle::Tensor> &rot, const std::vector<float> &voxel_size,
    const std::vector<float> &point_cloud_range, const std::vector<float> &post_center_range,
    const std::vector<int> &num_classes, const int down_ratio, const float score_threshold,
    const float nms_iou_threshold, const int nms_pre_max_size, const int nms_post_max_size, const bool with_velocity) {
  if (!hm[0].is_gpu()) PD_THROW("Unsupported device type for centerpoint postprocess operator.");
  PD_CHECK(hm[0].shape()[0] == 1, "hm[0] batch size must be 1.");
  const int T = static_cast<int>(hm.size());
  const int H = static_cast<int>(hm[0].shape()[2]), W = static_cast<int>(hm[0].shape()[3]);
  std::vector<const float *> p[6];
  std::vector<int32_t> hm_c(T);
  const std::vector<paddle::Tensor> *lists[6] = {&hm, &reg, &height, &dim, &vel, &rot};
  for (int k = 0; k < 6; ++k)
    for (int t = 0; t < T; ++t) p[k].push_back((*lists[k])[t].data<float>());
  for (int t = 0; t < T; ++t) hm_c[t] = static_cast<int32_t>(hm[t].shape()[1]);
  const int dims = with_velocity ? 9 : 7;
  const int rows = T * (nms_post_max_size > 1 ? nms_post_max_size : 1);
  auto bboxes = paddle::empty({rows, dims}, paddle::DataType::FLOAT32, paddle::GPUPlace());
  auto scores = paddle::empty({rows}, paddle::DataType::FLOAT32, paddle::GPUPlace());
  auto labels = paddle::empty({rows}, paddle::DataType::INT64, paddle::GPUPlace());
  auto counts = paddle::empty({T + 1}, paddle::DataType::INT32, paddle::GPUPlace());
  const size_t ws_bytes = p3d_centerpoint_postprocess_workspace_bytes(T, H, W, nms_pre_max_size, nms_post_max_size);
  auto ws = workspace(ws_bytes);
  P3D_CALL(p3d_centerpoint_postprocess(T, p[0].data(), hm_c.data(), p[1].data(), p[2].data(), p[3].data(), p[4].data(),
                                       p[5].data(), H, W, voxel_size.data(), point_cloud_range.data(),
                                       post_center_range.data(), num_classes.data(), down_ratio, score_threshold,
                                       nms_iou_threshold, nms_pre_max_size, nms_post_max_size, with_velocity ? 1 : 0,
                                       bboxes.data<float>(), scores.data<float>(), labels.data<int64_t>(),
                                       counts.data<int>(), ws.data<uint8_t>(), ws_bytes, hm[0].stream()));
  // the op's outputs have data-dependent shape {-1, 9|7}: one scalar read gives K, then slice
  const int k = counts.copy_to(paddle::CPUPlace(), true).data<int>()[T];
  return {paddle::experimental::slice(bboxes, {0}, {0}, {k}, {}, {}), paddle::experimental::slice(scores, {0}, {0}, {k}, {}, {}),
          paddle::experimental::slice(labels, {0}, {0}, {k}, {}, {})};
}

std::vector<std::vector<int64_t>> PostProcessInferShape(
    const std::vector<std::vector<int64_t>> &hm_shape, const std::vector<std::vector<int64_t>> &reg_shape,
    const std::vector<std::vector<int64_t>> &height_shape, const std::vector<std::vector<int64_t>> &dim_shape,
    const std::vector<std::vector<int64_t>> &vel_shape, const std::vector<std::vector<int64_t>> &rot_shape,
    const std::vector<float> &voxel_size, const std::vector<float> &point_cloud_range,
    const std::vector<float> &post_center_range, const std::vector<int> &num_classes, const int down_ratio,
    const float score_threshold, const float nms_iou_threshold, const int nms_pre_max_size,
    const int nms_post_max_size, const bool with_velocity) {
  if (with_velocity) return {{-1, 9}, {-1}, {-1}};
  return {{-1, 7}, {-1}, {-1}};
}

std::vector<paddle::DataType> PostProcessInferDtype(
    const std::vector<paddle::DataType> &hm_dtype, const std::vector<paddle::DataType> &reg_dtype,
    const std::vector<paddle::DataType> &height_dtype, const std::vector<paddle::DataType> &dim_dtype,
    const std::vector<paddle::DataType> &vel_dtype, const std::vector<paddle::DataType> &rot_dtype) {
  return {reg_dtype[0], hm_dtype[0], paddle::DataType::INT64};
}

PD_BUILD_OP(centerpoint_postprocess)
    .Inputs({paddle::Vec("HM"), paddle::Vec("REG"), paddle::Vec("HEIGHT"), paddle::Vec("DIM"), paddle::Vec("VEL"),
             paddle::Vec("ROT")})
    .Outputs({"BBOXES", "SCORES", "LABELS"})
    .SetKernelFn(PD_KERNEL(centerpoint_postprocess))
    .Attrs({"voxel_size: std::vector<float>", "point_cloud_range: std::vector<float>",
            "post_center_range: std::vector<float>", "num_classes: std::vector<int>", "down_ratio: int",
            "score_threshold: float", "nms_iou_threshold: float", "nms_pre_max_size: int", "nms_post_max_size: int",
            "with_velocity: bool"})
    .SetInferShapeFn(PD_INFER_SHAPE(PostProcessInferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(PostProcessInferDtype));

// ---------------------------------------------------------------- bev_pool_v2 / bev_pool_v2_bkwd
std::vector<paddle::Tensor> bev_pool_v2_forward(const paddle::Tensor &_depth, const paddle::Tensor &_feat,
                                                const paddle::Tensor &_ranks_depth, const paddle::Tensor &_ranks_feat,
                                                const paddle::Tensor &_ranks_bev, const paddle::Tensor &_interval_lengths,
                                                const paddle::Tensor &_interval_starts,
                                                const std::vector<int> &_bev_feat_shape) {
  P3D_CHECK_GPU(_feat);
  const int c = static_cast<int>(_feat.shape()[3]);
  const int n_intervals = static_cast<int>(_interval_lengths.shape()[0]);
  std::vector<int64_t> shape(_bev_feat_shape.begin(), _bev_feat_shape.end());
  auto out = paddle::empty(shape, _feat.type(), paddle::GPUPlace());  // zero-filled by the kernel's own memset
  P3D_CALL(p3d_bev_pool_v2(_depth.data<float>(), _feat.data<float>(), _ranks_depth.data<int>(), _ranks_feat.data<int>(),
                           _ranks_bev.data<int>(), _interval_lengths.data<int>(), _interval_starts.data<int>(),
                           n_intervals, c, out.data<float>(), out.numel(), _feat.stream()));
  return {out};
}

std::vector<paddle::Tensor> bev_pool_v2_backward(const paddle::Tensor &_out_grad, const paddle::Tensor &_depth,
                                                 const paddle::Tensor &_feat, const paddle::Tensor &_ranks_depth,
                                                 const paddle::Tensor &_ranks_feat, const paddle::Tensor &_ranks_bev,
                                                 const paddle::Tensor &_interval_lengths,
                                                 const paddle::Tensor &_interval_starts) {
  P3D_CHECK_GPU(_out_grad);
  const int c = static_cast<int>(_out_grad.shape()[3]);
  const int n_intervals = static_cast<int>(_interval_lengths.shape()[0]);
  auto depth_grad = paddle::empty(_depth.shape(), _depth.type(), paddle::GPUPlace());
  auto feat_grad = paddle::empty(_feat.shape(), _feat.type(), paddle::GPUPlace());
  P3D_CALL(p3d_bev_pool_v2_bkwd(_out_grad.data<float>(), _depth.data<float>(), _feat.data<float>(),
                                _ranks_depth.data<int>(), _ranks_feat.data<int>(), _ranks_bev.data<int>(),
                                _interval_lengths.data<int>(), _interval_starts.data<int>(), n_intervals, c,
                                depth_grad.data<float>(), depth_grad.numel(), feat_grad.data<float>(), feat_grad.numel(),
                                _out_grad.stream()));
  return {depth_grad, feat_grad};
}

std::vector<std::vector<int64_t>> BevPoolV2InferShape(std::vector<int64_t> a, std::vector<int64_t> b, std::vector<int64_t> c,
                                                      std::vector<int64_t> d, std::vector<int64_t> e, std::vector<int64_t> f,
                                                      std::vector<int64_t> g, const std::vector<int> _bev_feat_shape) {
  return {{_bev_feat_shape[0], _bev_feat_shape[1], _bev_feat_shape[2], _bev_feat_shape[3]}};
}
std::vector<paddle::DataType> BevPoolV2InferDtype(paddle::DataType a, paddle::DataType feat, paddle::DataType c,
                                                  paddle::DataType d, paddle::DataType e, paddle::DataType f,
                                                  paddle::DataType g) {
  return {feat};
}

PD_BUILD_OP(bev_pool_v2)
    .Inputs({"_depth", "_feat", "_ranks_depth", "_ranks_feat", "_ranks_bev", "_interval_lengths", "_interval_starts"})
    .Attrs({"_bev_feat_shape: std::vector<int>"})
    .Outputs({"out"})
    .SetKernelFn(PD_KERNEL(bev_pool_v2_forward))
    .SetInferShapeFn(PD_INFER_SHAPE(BevPoolV2InferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(BevPoolV2InferDtype));

std::vector<std::vector<int64_t>> BevPoolV2BkwdInferShape(std::vector<int64_t> og, std::vector<int64_t> depth,
                                                          std::vector<int64_t> feat, std::vector<int64_t> d,
                                                          std::vector<int64_t> e, std::vector<int64_t> f,
                                                          std::vector<int64_t> g, std::vector<int64_t> h) {
  return {depth, feat};
}
std::vector<paddle::DataType> BevPoolV2BkwdInferDtype(paddle::DataType og, paddle::DataType depth, paddle::DataType feat,
                                                      paddle::DataType d, paddle::DataType e, paddle::DataType f,
                                                      paddle::DataType g, paddle::DataType h) {
  return {depth, feat};
}

PD_BUILD_OP(bev_pool_v2_bkwd)
    .Inputs({"_out_grad", "_depth", "_feat", "_ranks_depth", "_ranks_feat", "_ranks_bev", "_interval_lengths",
             "_interval_starts"})
    .Outputs({"_depth_grad", "_feat_grad"})
    .SetKernelFn(PD_KERNEL(bev_pool_v2_backward))
    .SetInferShapeFn(PD_INFER_SHAPE(BevPoolV2BkwdInferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(BevPoolV2BkwdInferDtype));

// =====================================================================================================================
// Ops that have no custom-op counterpart in the reference because their arithmetic lives inside PaddlePaddle
// (paddle.sparse.nn.SubmConv3D / Conv3D / BatchNorm / ReLU, paddle.scatter, paddle.nn.Conv2D): new op names, same
// registration style.  paddle3d_b200/ops/sparse_nn.py and dense_head.py are the Python layer mirrors that call the
// same C entry points through ctypes.
// =====================================================================================================================

// ---------------------------------------------------------------- p3d_scatter_dense  (pillar_scatter.py:57-105, sparse_resnet.py:202-206)
std::vector<paddle::Tensor> p3d_scatter_dense_op(const paddle::Tensor &feats, const paddle::Tensor &coords,
                                                 const paddle::Tensor &num, const int batch, const int D, const int ny,
                                                 const int nx, const int use_z) {
  P3D_CHECK_GPU(feats);
  const int n = static_cast<int>(feats.shape()[0]), C = static_cast<int>(feats.shape()[1]);
  auto out = paddle::empty({batch, static_cast<int64_t>(C) * D, ny, nx}, paddle::DataType::FLOAT32, paddle::GPUPlace());
  const size_t ws_bytes = p3d_scatter_dense_workspace_bytes(batch, D, ny, nx);
  auto ws = workspace(ws_bytes);
  P3D_CALL(p3d_scatter_dense(feats.data<float>(), coords.data<int>(), num.data<int>(), n, C, batch, D, ny, nx, use_z,
                             out.data<float>(), ws.data<uint8_t>(), ws_bytes, feats.stream()));
  return {out};
}
std::vector<std::vector<int64_t>> ScatterInferShape(std::vector<int64_t> f, std::vector<int64_t> c, std::vector<int64_t> n,
                                                    const int &batch, const int &D, const int &ny, const int &nx,
                                                    const int &use_z) {
  return {{batch, f[1] * D, ny, nx}};
}
std::vector<paddle::DataType> ScatterInferDtype(paddle::DataType f, paddle::DataType c, paddle::DataType n) { return {f}; }

PD_BUILD_OP(p3d_scatter_dense)
    .Inputs({"FEATS", "COORDS", "NUM"})
    .Outputs({"OUT"})
    .Attrs({"batch: int", "D: int", "ny: int", "nx: int", "use_z: int"})
    .SetKernelFn(PD_KERNEL(p3d_scatter_dense_op))
    .SetInferShapeFn(PD_INFER_SHAPE(ScatterInferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(ScatterInferDtype));

// ---------------------------------------------------------------- rulebooks  (sparse_resnet.py:31-60: SubmConv3D / Conv3D site logic)
std::vector<paddle::Tensor> p3d_subm_rulebook_op(const paddle::Tensor &coords, const paddle::Tensor &num, const int batch,
                                                 const std::vector<int> &spatial, const std::vector<int> &ksize) {
  P3D_CHECK_GPU(coords);
  const int64_t cap = coords.shape()[0];
  const int64_t K = static_cast<int64_t>(ksize[0]) * ksize[1] * ksize[2];
  auto nbr = paddle::empty({cap, K}, paddle::DataType::INT32, paddle::GPUPlace());
  const size_t ws_bytes = p3d_sparse_rulebook_workspace_bytes(cap, cap);
  auto ws = workspace(ws_bytes);
  P3D_CALL(p3d_sparse_rulebook_subm(coords.data<int>(), num.data<int>(), cap, batch, spatial.data(), ksize.data(),
                                    nbr.data<int>(), ws.data<uint8_t>(), ws_bytes, coords.stream()));
  return {nbr};
}
std::vector<std::vector<int64_t>> SubmRbInferShape(std::vector<int64_t> c, std::vector<int64_t> n, const int &batch,
                                                   const std::vector<int> &spatial, const std::vector<int> &ksize) {
  return {{c[0], static_cast<int64_t>(ksize[0]) * ksize[1] * ksize[2]}};
}
std::vector<paddle::DataType> SubmRbInferDtype(paddle::DataType c, paddle::DataType n) { return {paddle::DataType::INT32}; }

PD_BUILD_OP(p3d_sparse_subm_rulebook)
    .Inputs({"COORDS", "NUM"})
    .Outputs({"NBR"})
    .Attrs({"batch: int", "spatial: std::vector<int>", "ksize: std::vector<int>"})
    .SetKernelFn(PD_KERNEL(p3d_subm_rulebook_op))
    .SetInferShapeFn(PD_INFER_SHAPE(SubmRbInferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(SubmRbInferDtype));

std::vector<paddle::Tensor> p3d_conv_rulebook_op(const paddle::Tensor &coords, const paddle::Tensor &num, const int batch,
                                                 const std::vector<int> &spatial, const std::vector<int> &ksize,
                                                 const std::vector<int> &stride, const std::vector<int> &padding,
                                                 const int out_cap) {
  P3D_CHECK_GPU(coords);
  const int64_t cap = coords.shape()[0];
  const int64_t K = static_cast<int64_t>(ksize[0]) * ksize[1] * ksize[2];
  auto out_coords = paddle::empty({out_cap, 4}, paddle::DataType::INT32, paddle::GPUPlace());
  auto n_out = paddle::empty({4}, paddle::DataType::INT32, paddle::GPUPlace());  // [count, .., .., table-full flag]
  auto nbr = paddle::empty({out_cap, K}, paddle::DataType::INT32, paddle::GPUPlace());
  const size_t ws_bytes = p3d_sparse_rulebook_workspace_bytes(cap, out_cap);
  auto ws = workspace(ws_bytes);
  P3D_CALL(p3d_sparse_rulebook_conv(coords.data<int>(), num.data<int>(), cap, batch, spatial.data(), ksize.data(),
                                    stride.data(), padding.data(), out_coords.data<int>(), n_out.data<int>(), out_cap,
                                    nbr.data<int>(), ws.data<uint8_t>(), ws_bytes, coords.stream()));
  return {out_coords, n_out, nbr};
}
std::vector<std::vector<int64_t>> ConvRbInferShape(std::vector<int64_t> c, std::vector<int64_t> n, const int &batch,
                                                   const std::vector<int> &spatial, const std::vector<int> &ksize,
                                                   const std::vector<int> &stride, const std::vector<int> &padding,
                                                   const int &out_cap) {
  return {{out_cap, 4}, {4}, {out_cap, static_cast<int64_t>(ksize[0]) * ksize[1] * ksize[2]}};
}
std::vector<paddle::DataType> ConvRbInferDtype(paddle::DataType c, paddle::DataType n) {
  return {paddle::DataType::INT32, paddle::DataType::INT32, paddle::DataType::INT32};
}

PD_BUILD_OP(p3d_sparse_conv_rulebook)
    .Inputs({"COORDS", "NUM"})
    .Outputs({"OUT_COORDS", "OUT_NUM", "NBR"})
    .Attrs({"batch: int", "spatial: std::vector<int>", "ksize: std::vector<int>", "stride: std::vector<int>",
            "padding: std::vector<int>", "out_cap: int"})
    .SetKernelFn(PD_KERNEL(p3d_conv_rulebook_op))
    .SetInferShapeFn(PD_INFER_SHAPE(ConvRbInferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(ConvRbInferDtype));

// ---------------------------------------------------------------- fused gather-GEMM (+ BN affine + residual + ReLU)
// RESIDUAL may be a 1-element tensor meaning "none" (Paddle custom ops of this API level have no optional inputs).
std::vector<paddle::Tensor> p3d_gather_gemm_op(const paddle::Tensor &in, const paddle::Tensor &nbr, const paddle::Tensor &num,
                                               const paddle::Tensor &weight, const paddle::Tensor &scale,
                                               const paddle::Tensor &shift, const paddle::Tensor &residual, const int relu,
                                               const int precision) {
  P3D_CHECK_GPU(in);
  const int64_t cap = nbr.shape()[0];
  const int K = static_cast<int>(nbr.shape()[1]);
  const int Cin = static_cast<int>(in.shape()[1]);
  const int Cout = static_cast<int>(weight.shape()[weight.shape().size() - 1]);  // [kD, kH, kW, Cin, Cout]
  auto out = paddle::empty({cap, Cout}, paddle::DataType::FLOAT32, paddle::GPUPlace());
  const float *res = residual.numel() > 1 ? residual.data<float>() : nullptr;
  P3D_CALL(p3d_sparse_conv_gather_gemm(in.data<float>(), nbr.data<int>(), num.data<int>(), cap, K, Cin, Cout,
                                       weight.data<float>(), scale.data<float>(), shift.data<float>(), res, relu,
                                       precision, out.data<float>(), in.stream()));
  return {out};
}
std::vector<std::vector<int64_t>> GgInferShape(std::vector<int64_t> in, std::vector<int64_t> nbr, std::vector<int64_t> num,
                                               std::vector<int64_t> w, std::vector<int64_t> sc, std::vector<int64_t> sh,
                                               std::vector<int64_t> res, const int &relu, const int &precision) {
  return {{nbr[0], w[w.size() - 1]}};
}
std::vector<paddle::DataType> GgInferDtype(paddle::DataType in, paddle::DataType nbr, paddle::DataType num, paddle::DataType w,
                                           paddle::DataType sc, paddle::DataType sh, paddle::DataType res) {
  return {in};
}

PD_BUILD_OP(p3d_sparse_gather_gemm)
    .Inputs({"IN", "NBR", "NUM", "WEIGHT", "SCALE", "SHIFT", "RESIDUAL"})
    .Outputs({"OUT"})
    .Attrs({"relu: int", "precision: int"})
    .SetKernelFn(PD_KERNEL(p3d_gather_gemm_op))
    .SetInferShapeFn(PD_INFER_SHAPE(GgInferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(GgInferDtype));

// ---------------------------------------------------------------- round 2: fp16-pair tensor-core paths + rank preparation
// Activations travel between these ops as FLOAT16 tensors holding (hi, lo') pairs ([rows, 2 * C], see include/p3d_b200.h);
// STATUS is a 1-element INT32 tensor the kernels OR range-overflow bits into (checked by the caller once per frame).
std::vector<paddle::Tensor> p3d_rows_to_h16_op(const paddle::Tensor &rows, const paddle::Tensor &num, const paddle::Tensor &status) {
  P3D_CHECK_GPU(rows);
  const int64_t cap = rows.shape()[0];
  const int C = static_cast<int>(rows.shape()[1]);
  auto out = paddle::empty({cap, 2 * C}, paddle::DataType::FLOAT16, paddle::GPUPlace());
  P3D_CALL(p3d_rows_convert_h16(rows.data<float>(), 1, num.data<int>(), cap, C, out.data(), const_cast<int *>(status.data<int>()),
                                rows.stream()));
  return {out};
}
std::vector<std::vector<int64_t>> ToH16InferShape(std::vector<int64_t> r, std::vector<int64_t> n, std::vector<int64_t> s) {
  return {{r[0], 2 * r[1]}};
}
std::vector<paddle::DataType> ToH16InferDtype(paddle::DataType r, paddle::DataType n, paddle::DataType s) {
  return {paddle::DataType::FLOAT16};
}
PD_BUILD_OP(p3d_rows_to_h16)
    .Inputs({"ROWS", "NUM", "STATUS"})
    .Outputs({"OUT"})
    .SetKernelFn(PD_KERNEL(p3d_rows_to_h16_op))
    .SetInferShapeFn(PD_INFER_SHAPE(ToH16InferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(ToH16InferDtype));

// sparse conv (SubmConv3D / Conv3D + BatchNorm(eval) + add + ReLU, sparse_resnet.py:31-60,84-111) on fp16-pair rows.
// WEIGHT is the packed image of p3d_sparse_conv_f16_pack_weights; RESIDUAL may be a 1-element tensor meaning "none";
// want_f32 = 1 returns fp32 rows [cap, Cout] (last layer before to_dense), else fp16-pair rows [cap, 2 * Cout].
std::vector<paddle::Tensor> p3d_sparse_conv_f16_op(const paddle::Tensor &in, const paddle::Tensor &nbr, const paddle::Tensor &num,
                                                   const paddle::Tensor &weight, const paddle::Tensor &scale,
                                                   const paddle::Tensor &shift, const paddle::Tensor &residual,
                                                   const paddle::Tensor &status, const int cin, const int cout, const int relu,
                                                   const int want_f32, const int max_splits) {
  P3D_CHECK_GPU(in);
  const int64_t cap = nbr.shape()[0];
  const int K = static_cast<int>(nbr.shape()[1]);
  auto out = want_f32 ? paddle::empty({cap, cout}, paddle::DataType::FLOAT32, paddle::GPUPlace())
                      : paddle::empty({cap, 2 * cout}, paddle::DataType::FLOAT16, paddle::GPUPlace());
  const size_t ws_bytes = p3d_sparse_conv_f16_workspace_bytes(cap, cout, max_splits);
  // the ticket head of the workspace must be zero on first use: paddle::full, not empty
  auto ws = paddle::full({static_cast<int64_t>(ws_bytes ? ws_bytes : 16)}, 0, paddle::DataType::UINT8, paddle::GPUPlace());
  const void *res = residual.numel() > 1 ? residual.data() : nullptr;
  P3D_CALL(p3d_sparse_conv_f16(in.data(), nbr.data<int>(), num.data<int>(), cap, K, cin, cout, weight.data(), scale.data<float>(),
                               shift.data<float>(), res, relu, want_f32 ? out.data<float>() : nullptr,
                               want_f32 ? nullptr : out.data(), ws_bytes ? ws.data<uint8_t>() : nullptr, ws_bytes, max_splits,
                               const_cast<int *>(status.data<int>()), in.stream()));
  return {out};
}
std::vector<std::vector<int64_t>> ScF16InferShape(std::vector<int64_t> in, std::vector<int64_t> nbr, std::vector<int64_t> num,
                                                  std::vector<int64_t> w, std::vector<int64_t> sc, std::vector<int64_t> sh,
                                                  std::vector<int64_t> res, std::vector<int64_t> st, const int &cin,
                                                  const int &cout, const int &relu, const int &want_f32, const int &max_splits) {
  return {{nbr[0], want_f32 ? static_cast<int64_t>(cout) : static_cast<int64_t>(2 * cout)}};
}
std::vector<paddle::DataType> ScF16InferDtype(paddle::DataType in, paddle::DataType nbr, paddle::DataType num, paddle::DataType w,
                                              paddle::DataType sc, paddle::DataType sh, paddle::DataType res, paddle::DataType st) {
  return {in};  // refined at run time by want_f32 (attrs are not visible to the dtype function of this API level)
}
PD_BUILD_OP(p3d_sparse_conv_f16)
    .Inputs({"IN", "NBR", "NUM", "WEIGHT", "SCALE", "SHIFT", "RESIDUAL", "STATUS"})
    .Outputs({"OUT"})
    .Attrs({"cin: int", "cout: int", "relu: int", "want_f32: int", "max_splits: int"})
    .SetKernelFn(PD_KERNEL(p3d_sparse_conv_f16_op))
    .SetInferShapeFn(PD_INFER_SHAPE(ScF16InferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(ScF16InferDtype));

// The same layer on the narrow-layer warp-MMA kernel (csrc/sparse_conv_wm.cu): (cin, cout) in {(16,16), (16,32), (32,32)}.
// WEIGHT is the packed image of p3d_sparse_conv_wm_pack_weights; everything else as p3d_sparse_conv_f16.
std::vector<paddle::Tensor> p3d_sparse_conv_wm_op(const paddle::Tensor &in, const paddle::Tensor &nbr, const paddle::Tensor &num,
                                                  const paddle::Tensor &weight, const paddle::Tensor &scale,
                                                  const paddle::Tensor &shift, const paddle::Tensor &residual,
                                                  const paddle::Tensor &status, const int cin, const int cout, const int relu,
                                                  const int want_f32) {
  P3D_CHECK_GPU(in);
  const int64_t cap = nbr.shape()[0];
  const int K = static_cast<int>(nbr.shape()[1]);
  auto out = want_f32 ? paddle::empty({cap, cout}, paddle::DataType::FLOAT32, paddle::GPUPlace())
                      : paddle::empty({cap, 2 * cout}, paddle::DataType::FLOAT16, paddle::GPUPlace());
  const size_t ws_bytes = p3d_sparse_conv_wm_workspace_bytes(cap, cout);
  // the ticket head of the workspace must be zero on first use: paddle::full, not empty
  auto ws = paddle::full({static_cast<int64_t>(ws_bytes ? ws_bytes : 16)}, 0, paddle::DataType::UINT8, paddle::GPUPlace());
  const void *res = residual.numel() > 1 ? residual.data() : nullptr;
  P3D_CALL(p3d_sparse_conv_wm(in.data(), nbr.data<int>(), num.data<int>(), cap, K, cin, cout, weight.data(), scale.data<float>(),
                              shift.data<float>(), res, relu, want_f32 ? out.data<float>() : nullptr,
                              want_f32 ? nullptr : out.data(), ws.data<uint8_t>(), ws_bytes,
                              const_cast<int *>(status.data<int>()), in.stream()));
  return {out};
}
std::vector<std::vector<int64_t>> ScWmInferShape(std::vector<int64_t> in, std::vector<int64_t> nbr, std::vector<int64_t> num,
                                                 std::vector<int64_t> w, std::vector<int64_t> sc, std::vector<int64_t> sh,
                                                 std::vector<int64_t> res, std::vector<int64_t> st, const int &cin,
                                                 const int &cout, const int &relu, const int &want_f32) {
  return {{nbr[0], want_f32 ? static_cast<int64_t>(cout) : static_cast<int64_t>(2 * cout)}};
}
PD_BUILD_OP(p3d_sparse_conv_wm)
    .Inputs({"IN", "NBR", "NUM", "WEIGHT", "SCALE", "SHIFT", "RESIDUAL", "STATUS"})
    .Outputs({"OUT"})
    .Attrs({"cin: int", "cout: int", "relu: int", "want_f32: int"})
    .SetKernelFn(PD_KERNEL(p3d_sparse_conv_wm_op))
    .SetInferShapeFn(PD_INFER_SHAPE(ScWmInferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(ScF16InferDtype));

// dense Conv2D / Conv2DTranspose + BatchNorm2D(eval) + ReLU on pixel fp16-pair rows (second_backbone.py:72-120,
// second_fpn.py:99-160, center_head.py:43-220).  IMAGE [B*H*W, 2*Cin] FLOAT16; WEIGHT = packed image
// (p3d_dense_conv2d_f16_pack_weights per N tile).  Output rows have out_channels channels, this layer writes
// [out_c0, out_c0 + cout) (channel concat of the neck for free).
std::vector<paddle::Tensor> p3d_dense_conv2d_f16_op(const paddle::Tensor &image, const paddle::Tensor &weight,
                                                    const paddle::Tensor &scale, const paddle::Tensor &shift,
                                                    const paddle::Tensor &status, const std::vector<int> &bhwc, const int cout,
                                                    const int n_tile, const int kernel, const int stride, const int pad,
                                                    const int up, const int relu, const int out_channels, const int out_c0) {
  P3D_CHECK_GPU(image);
  const int B = bhwc[0], H = bhwc[1], W = bhwc[2], Cin = bhwc[3];
  const int oH = up > 1 ? H * up : (H + 2 * pad - kernel) / stride + 1, oW = up > 1 ? W * up : (W + 2 * pad - kernel) / stride + 1;
  auto out = paddle::empty({static_cast<int64_t>(B) * oH * oW, 2 * out_channels}, paddle::DataType::FLOAT16, paddle::GPUPlace());
  const int k = up > 1 ? up : kernel, s = up > 1 ? up : stride;
  P3D_CALL(p3d_dense_conv2d_f16(image.data(), B, H, W, Cin, weight.data(), cout, n_tile, k, k, s, up > 1 ? 0 : pad, up,
                                scale.data<float>(), shift.data<float>(), relu, out.data(), out_channels, out_c0, nullptr, 0, 0,
                                const_cast<int *>(status.data<int>()), image.stream()));
  return {out};
}
std::vector<std::vector<int64_t>> DcF16InferShape(std::vector<int64_t> im, std::vector<int64_t> w, std::vector<int64_t> sc,
                                                  std::vector<int64_t> sh, std::vector<int64_t> st, const std::vector<int> &bhwc,
                                                  const int &cout, const int &n_tile, const int &kernel, const int &stride,
                                                  const int &pad, const int &up, const int &relu, const int &out_channels,
                                                  const int &out_c0) {
  const int64_t oH = up > 1 ? bhwc[1] * up : (bhwc[1] + 2 * pad - kernel) / stride + 1;
  const int64_t oW = up > 1 ? bhwc[2] * up : (bhwc[2] + 2 * pad - kernel) / stride + 1;
  return {{bhwc[0] * oH * oW, 2 * static_cast<int64_t>(out_channels)}};
}
std::vector<paddle::DataType> DcF16InferDtype(paddle::DataType im, paddle::DataType w, paddle::DataType sc, paddle::DataType sh,
                                              paddle::DataType st) {
  return {paddle::DataType::FLOAT16};
}
PD_BUILD_OP(p3d_dense_conv2d_f16)
    .Inputs({"IMAGE", "WEIGHT", "SCALE", "SHIFT", "STATUS"})
    .Outputs({"OUT"})
    .Attrs({"bhwc: std::vector<int>", "cout: int", "n_tile: int", "kernel: int", "stride: int", "pad: int", "up: int",
            "relu: int", "out_channels: int", "out_c0: int"})
    .SetKernelFn(PD_KERNEL(p3d_dense_conv2d_f16_op))
    .SetInferShapeFn(PD_INFER_SHAPE(DcF16InferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(DcF16InferDtype));

// LSSViewTransformer.voxel_pooling_prepare_v2 (bevdet_transformer.py:230-274) as an op: COOR [B, N, D, H, W, 3] ->
// five capacity-sized INT32 rank arrays + COUNTS {n_kept, n_intervals}; the Python wrapper slices them.
std::vector<paddle::Tensor> p3d_bev_pool_prepare_op(const paddle::Tensor &coor, const std::vector<float> &lower,
                                                    const std::vector<float> &interval, const std::vector<int> &grid_size) {
  P3D_CHECK_GPU(coor);
  const auto sh = coor.shape();
  const int B = sh[0], N = sh[1], D = sh[2], H = sh[3], W = sh[4];
  const int64_t n = static_cast<int64_t>(B) * N * D * H * W;
  std::vector<paddle::Tensor> out;
  for (int i = 0; i < 5; ++i) out.push_back(paddle::empty({n}, paddle::DataType::INT32, paddle::GPUPlace()));
  out.push_back(paddle::empty({2}, paddle::DataType::INT32, paddle::GPUPlace()));
  const size_t ws_bytes = p3d_bev_pool_prepare_workspace_bytes(n);
  auto ws = workspace(ws_bytes);
  P3D_CALL(p3d_bev_pool_prepare(coor.data<float>(), B, N, D, H, W, lower.data(), interval.data(), grid_size.data(),
                                out[0].data<int>(), out[1].data<int>(), out[2].data<int>(), out[3].data<int>(), out[4].data<int>(),
                                out[5].data<int>(), ws.data<uint8_t>(), ws_bytes, coor.stream()));
  return out;
}
std::vector<std::vector<int64_t>> PrepInferShape(std::vector<int64_t> c, const std::vector<float> &lower,
                                                 const std::vector<float> &interval, const std::vector<int> &grid_size) {
  const int64_t n = c[0] * c[1] * c[2] * c[3] * c[4];
  return {{n}, {n}, {n}, {n}, {n}, {2}};
}
std::vector<paddle::DataType> PrepInferDtype(paddle::DataType c) {
  return {paddle::DataType::INT32, paddle::DataType::INT32, paddle::DataType::INT32, paddle::DataType::INT32,
          paddle::DataType::INT32, paddle::DataType::INT32};
}
PD_BUILD_OP(p3d_bev_pool_prepare)
    .Inputs({"COOR"})
    .Outputs({"RANKS_BEV", "RANKS_DEPTH", "RANKS_FEAT", "INTERVAL_STARTS", "INTERVAL_LENGTHS", "COUNTS"})
    .Attrs({"grid_lower_bound: std::vector<float>", "grid_interval: std::vector<float>", "grid_size: std::vector<int>"})
    .SetKernelFn(PD_KERNEL(p3d_bev_pool_prepare_op))
    .SetInferShapeFn(PD_INFER_SHAPE(PrepInferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(PrepInferDtype));

// LSSViewTransformer.get_lidar_coor fused with voxel_pooling_prepare_v2: CAMS [B*N*24 + B*9] fp32 (the p3d_lss_camera
// entries, then bda [B, 3, 3]) and the frustum axes DEPTH [D], XS [W], YS [H] -> the outputs of p3d_bev_pool_prepare plus
// COOR: [B, N, D, H, W, 3] with with_coor (get_lidar_coor), otherwise an empty [0] tensor and no coordinate is written.
std::vector<paddle::Tensor> p3d_lss_prepare_op(const paddle::Tensor &cams, const paddle::Tensor &axis_d,
                                               const paddle::Tensor &axis_x, const paddle::Tensor &axis_y, int B, int N,
                                               const std::vector<float> &lower, const std::vector<float> &interval,
                                               const std::vector<int> &grid_size, bool with_coor) {
  P3D_CHECK_GPU(cams);
  const int D = axis_d.shape()[0], W = axis_x.shape()[0], H = axis_y.shape()[0];
  const int64_t n = static_cast<int64_t>(B) * N * D * H * W;
  std::vector<paddle::Tensor> out;
  for (int i = 0; i < 5; ++i) out.push_back(paddle::empty({n}, paddle::DataType::INT32, paddle::GPUPlace()));
  out.push_back(paddle::empty({2}, paddle::DataType::INT32, paddle::GPUPlace()));
  if (with_coor)
    out.push_back(paddle::empty({B, N, D, H, W, 3}, paddle::DataType::FLOAT32, paddle::GPUPlace()));
  else
    out.push_back(paddle::empty({0}, paddle::DataType::FLOAT32, paddle::GPUPlace()));
  const size_t ws_bytes = p3d_bev_pool_prepare_workspace_bytes(n);
  auto ws = workspace(ws_bytes);
  const float *c = cams.data<float>();
  P3D_CALL(p3d_lss_prepare(reinterpret_cast<const p3d_lss_camera *>(c), c + static_cast<int64_t>(B) * N * 24,
                           axis_d.data<float>(), axis_x.data<float>(), axis_y.data<float>(), B, N, D, H, W, lower.data(),
                           interval.data(), grid_size.data(), with_coor ? out[6].data<float>() : nullptr, out[0].data<int>(), out[1].data<int>(),
                           out[2].data<int>(), out[3].data<int>(), out[4].data<int>(), out[5].data<int>(), ws.data<uint8_t>(),
                           ws_bytes, cams.stream()));
  return out;
}
std::vector<std::vector<int64_t>> LssPrepInferShape(std::vector<int64_t> c, std::vector<int64_t> d, std::vector<int64_t> x,
                                                    std::vector<int64_t> y, int B, int N, const std::vector<float> &lower,
                                                    const std::vector<float> &interval, const std::vector<int> &grid_size,
                                                    bool with_coor) {
  const int64_t n = static_cast<int64_t>(B) * N * d[0] * y[0] * x[0];
  const std::vector<int64_t> coor = with_coor ? std::vector<int64_t>{B, N, d[0], y[0], x[0], 3} : std::vector<int64_t>{0};
  return {{n}, {n}, {n}, {n}, {n}, {2}, coor};
}
std::vector<paddle::DataType> LssPrepInferDtype(paddle::DataType c, paddle::DataType d, paddle::DataType x, paddle::DataType y) {
  return {paddle::DataType::INT32, paddle::DataType::INT32, paddle::DataType::INT32, paddle::DataType::INT32,
          paddle::DataType::INT32, paddle::DataType::INT32, paddle::DataType::FLOAT32};
}
PD_BUILD_OP(p3d_lss_prepare)
    .Inputs({"CAMS", "DEPTH", "XS", "YS"})
    .Outputs({"RANKS_BEV", "RANKS_DEPTH", "RANKS_FEAT", "INTERVAL_STARTS", "INTERVAL_LENGTHS", "COUNTS", "COOR"})
    .Attrs({"B: int", "N: int", "grid_lower_bound: std::vector<float>", "grid_interval: std::vector<float>",
            "grid_size: std::vector<int>", "with_coor: bool"})
    .SetKernelFn(PD_KERNEL(p3d_lss_prepare_op))
    .SetInferShapeFn(PD_INFER_SHAPE(LssPrepInferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(LssPrepInferDtype));

// bev_pool_v2 with the interval count on the device (COUNTS from p3d_bev_pool_prepare / p3d_lss_prepare) into
// view_transform's [B, Z * C, Y, X] layout; bzyx = (B, Z, Y, X).
std::vector<paddle::Tensor> p3d_bev_pool_v2_dev_op(const paddle::Tensor &depth, const paddle::Tensor &feat,
                                                   const paddle::Tensor &ranks_depth, const paddle::Tensor &ranks_feat,
                                                   const paddle::Tensor &ranks_bev, const paddle::Tensor &interval_lengths,
                                                   const paddle::Tensor &interval_starts, const paddle::Tensor &counts,
                                                   const std::vector<int> &bzyx) {
  P3D_CHECK_GPU(feat);
  const int c = feat.shape()[feat.shape().size() - 1];
  auto out = paddle::empty({bzyx[0], bzyx[1] * c, bzyx[2], bzyx[3]}, paddle::DataType::FLOAT32, paddle::GPUPlace());
  P3D_CALL(p3d_bev_pool_v2_dev(depth.data<float>(), feat.data<float>(), ranks_depth.data<int>(), ranks_feat.data<int>(),
                               ranks_bev.data<int>(), interval_lengths.data<int>(), interval_starts.data<int>(),
                               counts.data<int>(), ranks_bev.shape()[0], c, bzyx[0], bzyx[1], bzyx[2], bzyx[3], 1,
                               out.data<float>(), feat.stream()));
  return {out};
}
std::vector<std::vector<int64_t>> PoolDevInferShape(std::vector<int64_t> d, std::vector<int64_t> f, std::vector<int64_t> a,
                                                    std::vector<int64_t> b, std::vector<int64_t> e, std::vector<int64_t> g,
                                                    std::vector<int64_t> h, std::vector<int64_t> k, const std::vector<int> &bzyx) {
  return {{bzyx[0], bzyx[1] * f.back(), bzyx[2], bzyx[3]}};
}
std::vector<paddle::DataType> PoolDevInferDtype(paddle::DataType d, paddle::DataType f, paddle::DataType a, paddle::DataType b,
                                                paddle::DataType e, paddle::DataType g, paddle::DataType h, paddle::DataType k) {
  return {paddle::DataType::FLOAT32};
}
PD_BUILD_OP(p3d_bev_pool_v2_dev)
    .Inputs({"DEPTH", "FEAT", "RANKS_DEPTH", "RANKS_FEAT", "RANKS_BEV", "INTERVAL_LENGTHS", "INTERVAL_STARTS", "COUNTS"})
    .Outputs({"OUT"})
    .Attrs({"bzyx: std::vector<int>"})
    .SetKernelFn(PD_KERNEL(p3d_bev_pool_v2_dev_op))
    .SetInferShapeFn(PD_INFER_SHAPE(PoolDevInferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(PoolDevInferDtype));

// p3d_dense_conv2d_f16 with a residual added before ReLU (CustomResNet BasicBlock: relu(bn2(conv2(.)) + identity)):
// RESIDUAL [B*oH*oW, 2*res_channels] FLOAT16 pixel rows, channels [0, cout) added; H16 output, stride-1 or -2 conv.
std::vector<paddle::Tensor> p3d_dense_conv2d_f16_residual_op(const paddle::Tensor &image, const paddle::Tensor &weight,
                                                             const paddle::Tensor &scale, const paddle::Tensor &shift,
                                                             const paddle::Tensor &residual, const paddle::Tensor &status,
                                                             const std::vector<int> &bhwc, const int cout, const int n_tile,
                                                             const int kernel, const int stride, const int pad, const int relu,
                                                             const int out_channels, const int out_c0, const int res_channels) {
  P3D_CHECK_GPU(image);
  const int B = bhwc[0], H = bhwc[1], W = bhwc[2], Cin = bhwc[3];
  const int oH = (H + 2 * pad - kernel) / stride + 1, oW = (W + 2 * pad - kernel) / stride + 1;
  auto out = paddle::empty({static_cast<int64_t>(B) * oH * oW, 2 * out_channels}, paddle::DataType::FLOAT16, paddle::GPUPlace());
  P3D_CALL(p3d_dense_conv2d_f16_residual(image.data(), B, H, W, Cin, weight.data(), cout, n_tile, kernel, kernel, stride, pad, 1,
                                         scale.data<float>(), shift.data<float>(), relu, out.data(), out_channels, out_c0, nullptr,
                                         residual.data(), res_channels, 0, 0, const_cast<int *>(status.data<int>()),
                                         image.stream()));
  return {out};
}
std::vector<std::vector<int64_t>> DcF16ResInferShape(std::vector<int64_t> im, std::vector<int64_t> w, std::vector<int64_t> sc,
                                                     std::vector<int64_t> sh, std::vector<int64_t> res, std::vector<int64_t> st,
                                                     const std::vector<int> &bhwc, const int &cout, const int &n_tile,
                                                     const int &kernel, const int &stride, const int &pad, const int &relu,
                                                     const int &out_channels, const int &out_c0, const int &res_channels) {
  const int64_t oH = (bhwc[1] + 2 * pad - kernel) / stride + 1, oW = (bhwc[2] + 2 * pad - kernel) / stride + 1;
  return {{bhwc[0] * oH * oW, 2 * static_cast<int64_t>(out_channels)}};
}
std::vector<paddle::DataType> DcF16ResInferDtype(paddle::DataType im, paddle::DataType w, paddle::DataType sc,
                                                 paddle::DataType sh, paddle::DataType res, paddle::DataType st) {
  return {paddle::DataType::FLOAT16};
}
PD_BUILD_OP(p3d_dense_conv2d_f16_residual)
    .Inputs({"IMAGE", "WEIGHT", "SCALE", "SHIFT", "RESIDUAL", "STATUS"})
    .Outputs({"OUT"})
    .Attrs({"bhwc: std::vector<int>", "cout: int", "n_tile: int", "kernel: int", "stride: int", "pad: int", "relu: int",
            "out_channels: int", "out_c0: int", "res_channels: int"})
    .SetKernelFn(PD_KERNEL(p3d_dense_conv2d_f16_residual_op))
    .SetInferShapeFn(PD_INFER_SHAPE(DcF16ResInferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(DcF16ResInferDtype));

// nn.Upsample(scale_factor, mode='bilinear', align_corners=True) of FPN_LSS on pixel fp16-pair rows: IMAGE [B*h*w, 2*C]
// FLOAT16 -> [B*sh*sw, 2*out_channels] with channels [out_c0, out_c0 + C) written (the rest of a new tensor is left as
// allocated: callers that concatenate write the other channels).
std::vector<paddle::Tensor> p3d_upsample_bilinear_h16_op(const paddle::Tensor &image, const paddle::Tensor &status,
                                                         const std::vector<int> &bhwc, const int scale, const int out_channels,
                                                         const int out_c0) {
  P3D_CHECK_GPU(image);
  const int B = bhwc[0], h = bhwc[1], w = bhwc[2], C = bhwc[3];
  auto out = paddle::empty({static_cast<int64_t>(B) * h * scale * w * scale, 2 * out_channels}, paddle::DataType::FLOAT16,
                           paddle::GPUPlace());
  P3D_CALL(p3d_upsample_bilinear_h16(image.data(), B, h, w, C, scale, out.data(), out_channels, out_c0,
                                     const_cast<int *>(status.data<int>()), image.stream()));
  return {out};
}
std::vector<std::vector<int64_t>> UpH16InferShape(std::vector<int64_t> im, std::vector<int64_t> st, const std::vector<int> &bhwc,
                                                  const int &scale, const int &out_channels, const int &out_c0) {
  return {{static_cast<int64_t>(bhwc[0]) * bhwc[1] * scale * bhwc[2] * scale, 2 * static_cast<int64_t>(out_channels)}};
}
std::vector<paddle::DataType> UpH16InferDtype(paddle::DataType im, paddle::DataType st) { return {paddle::DataType::FLOAT16}; }
PD_BUILD_OP(p3d_upsample_bilinear_h16)
    .Inputs({"IMAGE", "STATUS"})
    .Outputs({"OUT"})
    .Attrs({"bhwc: std::vector<int>", "scale: int", "out_channels: int", "out_c0: int"})
    .SetKernelFn(PD_KERNEL(p3d_upsample_bilinear_h16_op))
    .SetInferShapeFn(PD_INFER_SHAPE(UpH16InferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(UpH16InferDtype));

// bev_pool_v2 with the interval count on the device straight into pixel fp16-pair rows [B*Y*X, 2*out_channels] FLOAT16
// (channel z * C + c of a cell; empty cells and channels >= Z * C zero), the first dense conv's input; bzyx = (B, Z, Y, X).
std::vector<paddle::Tensor> p3d_bev_pool_v2_dev_h16_op(const paddle::Tensor &depth, const paddle::Tensor &feat,
                                                       const paddle::Tensor &ranks_depth, const paddle::Tensor &ranks_feat,
                                                       const paddle::Tensor &ranks_bev, const paddle::Tensor &interval_lengths,
                                                       const paddle::Tensor &interval_starts, const paddle::Tensor &counts,
                                                       const paddle::Tensor &status, const std::vector<int> &bzyx,
                                                       const int out_channels) {
  P3D_CHECK_GPU(feat);
  const int c = feat.shape()[feat.shape().size() - 1];
  auto out = paddle::empty({static_cast<int64_t>(bzyx[0]) * bzyx[2] * bzyx[3], 2 * out_channels}, paddle::DataType::FLOAT16,
                           paddle::GPUPlace());
  P3D_CALL(p3d_bev_pool_v2_dev_h16(depth.data<float>(), feat.data<float>(), ranks_depth.data<int>(), ranks_feat.data<int>(),
                                   ranks_bev.data<int>(), interval_lengths.data<int>(), interval_starts.data<int>(),
                                   counts.data<int>(), ranks_bev.shape()[0], c, bzyx[0], bzyx[1], bzyx[2], bzyx[3], out.data(),
                                   out_channels, const_cast<int *>(status.data<int>()), feat.stream()));
  return {out};
}
std::vector<std::vector<int64_t>> PoolH16InferShape(std::vector<int64_t> d, std::vector<int64_t> f, std::vector<int64_t> a,
                                                    std::vector<int64_t> b, std::vector<int64_t> e, std::vector<int64_t> g,
                                                    std::vector<int64_t> h, std::vector<int64_t> k, std::vector<int64_t> st,
                                                    const std::vector<int> &bzyx, const int &out_channels) {
  return {{static_cast<int64_t>(bzyx[0]) * bzyx[2] * bzyx[3], 2 * static_cast<int64_t>(out_channels)}};
}
std::vector<paddle::DataType> PoolH16InferDtype(paddle::DataType d, paddle::DataType f, paddle::DataType a, paddle::DataType b,
                                                paddle::DataType e, paddle::DataType g, paddle::DataType h, paddle::DataType k,
                                                paddle::DataType st) {
  return {paddle::DataType::FLOAT16};
}
PD_BUILD_OP(p3d_bev_pool_v2_dev_h16)
    .Inputs({"DEPTH", "FEAT", "RANKS_DEPTH", "RANKS_FEAT", "RANKS_BEV", "INTERVAL_LENGTHS", "INTERVAL_STARTS", "COUNTS", "STATUS"})
    .Outputs({"OUT"})
    .Attrs({"bzyx: std::vector<int>", "out_channels: int"})
    .SetKernelFn(PD_KERNEL(p3d_bev_pool_v2_dev_h16_op))
    .SetInferShapeFn(PD_INFER_SHAPE(PoolH16InferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(PoolH16InferDtype));

// BEVDet4D's shift_feature on pixel fp16-pair rows: channels [0, C) of IMAGE [B*h*w, 2*in_C] FLOAT16 resampled by the
// per-sample affine TF [B, 6] FLOAT32 (ops.bev_pool_v2.pack_shift) into channels [out_c0, out_c0 + C) of a new
// [B*h*w, 2*out_channels] (the rest of the tensor is left as allocated: the concat's other channels come from
// pre_process).  bhwc = (B, h, w, in_C).
std::vector<paddle::Tensor> p3d_bev_shift_h16_op(const paddle::Tensor &image, const paddle::Tensor &tf,
                                                 const paddle::Tensor &status, const std::vector<int> &bhwc, const int C,
                                                 const int out_channels, const int out_c0) {
  P3D_CHECK_GPU(image);
  const int B = bhwc[0], h = bhwc[1], w = bhwc[2], in_C = bhwc[3];
  auto out = paddle::empty({static_cast<int64_t>(B) * h * w, 2 * out_channels}, paddle::DataType::FLOAT16, paddle::GPUPlace());
  P3D_CALL(p3d_bev_shift_h16(image.data(), B, h, w, in_C, C, tf.data<float>(), out.data(), out_channels, out_c0,
                             const_cast<int *>(status.data<int>()), image.stream()));
  return {out};
}
std::vector<std::vector<int64_t>> ShiftH16InferShape(std::vector<int64_t> im, std::vector<int64_t> tf, std::vector<int64_t> st,
                                                     const std::vector<int> &bhwc, const int &C, const int &out_channels,
                                                     const int &out_c0) {
  return {{static_cast<int64_t>(bhwc[0]) * bhwc[1] * bhwc[2], 2 * static_cast<int64_t>(out_channels)}};
}
std::vector<paddle::DataType> ShiftH16InferDtype(paddle::DataType im, paddle::DataType tf, paddle::DataType st) {
  return {paddle::DataType::FLOAT16};
}
PD_BUILD_OP(p3d_bev_shift_h16)
    .Inputs({"IMAGE", "TF", "STATUS"})
    .Outputs({"OUT"})
    .Attrs({"bhwc: std::vector<int>", "C: int", "out_channels: int", "out_c0: int"})
    .SetKernelFn(PD_KERNEL(p3d_bev_shift_h16_op))
    .SetInferShapeFn(PD_INFER_SHAPE(ShiftH16InferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(ShiftH16InferDtype));

// ---------------------------------------------------------------- p3d_bevdet_postprocess  (BEVDet's CenterHead.get_bboxes, Python in the reference)
// nms_type: 0 rotate / 1 circle per task; nms_rescale_factor: one factor per class, the tasks' classes concatenated.
std::vector<paddle::Tensor> p3d_bevdet_postprocess_op(
    const std::vector<paddle::Tensor> &hm, const std::vector<paddle::Tensor> &reg,
    const std::vector<paddle::Tensor> &height, const std::vector<paddle::Tensor> &dim,
    const std::vector<paddle::Tensor> &vel, const std::vector<paddle::Tensor> &rot, const std::vector<float> &voxel_size,
    const std::vector<float> &point_cloud_range, const std::vector<float> &post_center_range,
    const std::vector<int> &label_offsets, const int out_size_factor, const float score_threshold, const int max_num,
    const int pre_max_size, const int post_max_size, const std::vector<int> &nms_type, const std::vector<float> &nms_thr,
    const std::vector<float> &min_radius, const std::vector<float> &nms_rescale_factor) {
  P3D_CHECK_GPU(hm[0]);
  PD_CHECK(hm[0].shape()[0] == 1, "hm[0] batch size must be 1.");
  const int T = static_cast<int>(hm.size());
  const int H = static_cast<int>(hm[0].shape()[2]), W = static_cast<int>(hm[0].shape()[3]);
  std::vector<const float *> p[6];
  std::vector<int32_t> hm_c(T);
  const std::vector<paddle::Tensor> *lists[6] = {&hm, &reg, &height, &dim, &vel, &rot};
  size_t classes = 0;
  for (int k = 0; k < 6; ++k) {
    PD_CHECK(static_cast<int>(lists[k]->size()) == T, "one tensor per task in every input list.");
    for (int t = 0; t < T; ++t) p[k].push_back((*lists[k])[t].data<float>());
  }
  for (int t = 0; t < T; ++t) classes += hm_c[t] = static_cast<int32_t>(hm[t].shape()[1]);
  PD_CHECK(static_cast<int>(label_offsets.size()) >= T && static_cast<int>(nms_type.size()) == T &&
               static_cast<int>(nms_thr.size()) == T && static_cast<int>(min_radius.size()) == T,
           "label_offsets, nms_type, nms_thr and min_radius have one entry per task.");
  PD_CHECK(nms_rescale_factor.size() == classes, "nms_rescale_factor has one entry per class.");
  const int rows = T * (post_max_size > 1 ? post_max_size : 1);
  auto bboxes = paddle::empty({rows, 9}, paddle::DataType::FLOAT32, paddle::GPUPlace());
  auto scores = paddle::empty({rows}, paddle::DataType::FLOAT32, paddle::GPUPlace());
  auto labels = paddle::empty({rows}, paddle::DataType::INT64, paddle::GPUPlace());
  auto counts = paddle::empty({T + 1}, paddle::DataType::INT32, paddle::GPUPlace());
  const size_t ws_bytes = p3d_bevdet_postprocess_workspace_bytes(T, hm_c.data(), H, W, max_num);
  auto ws = workspace(ws_bytes);
  P3D_CALL(p3d_bevdet_postprocess(T, p[0].data(), hm_c.data(), p[1].data(), p[2].data(), p[3].data(), p[4].data(),
                                  p[5].data(), H, W, voxel_size.data(), point_cloud_range.data(), post_center_range.data(),
                                  out_size_factor, score_threshold, max_num, pre_max_size, post_max_size, nms_type.data(),
                                  nms_thr.data(), min_radius.data(), nms_rescale_factor.data(), label_offsets.data(),
                                  bboxes.data<float>(), scores.data<float>(), labels.data<int64_t>(), counts.data<int>(),
                                  ws.data<uint8_t>(), ws_bytes, hm[0].stream()));
  // data-dependent shape {-1, 9}: one scalar read gives K, then slice
  const int k = counts.copy_to(paddle::CPUPlace(), true).data<int>()[T];
  return {paddle::experimental::slice(bboxes, {0}, {0}, {k}, {}, {}), paddle::experimental::slice(scores, {0}, {0}, {k}, {}, {}),
          paddle::experimental::slice(labels, {0}, {0}, {k}, {}, {})};
}

std::vector<std::vector<int64_t>> BevdetPostProcessInferShape(
    const std::vector<std::vector<int64_t>> &hm_shape, const std::vector<std::vector<int64_t>> &reg_shape,
    const std::vector<std::vector<int64_t>> &height_shape, const std::vector<std::vector<int64_t>> &dim_shape,
    const std::vector<std::vector<int64_t>> &vel_shape, const std::vector<std::vector<int64_t>> &rot_shape) {
  return {{-1, 9}, {-1}, {-1}};
}

PD_BUILD_OP(p3d_bevdet_postprocess)
    .Inputs({paddle::Vec("HM"), paddle::Vec("REG"), paddle::Vec("HEIGHT"), paddle::Vec("DIM"), paddle::Vec("VEL"),
             paddle::Vec("ROT")})
    .Outputs({"BBOXES", "SCORES", "LABELS"})
    .SetKernelFn(PD_KERNEL(p3d_bevdet_postprocess_op))
    .Attrs({"voxel_size: std::vector<float>", "point_cloud_range: std::vector<float>",
            "post_center_range: std::vector<float>", "label_offsets: std::vector<int>", "out_size_factor: int",
            "score_threshold: float", "max_num: int", "pre_max_size: int", "post_max_size: int",
            "nms_type: std::vector<int>", "nms_thr: std::vector<float>", "min_radius: std::vector<float>",
            "nms_rescale_factor: std::vector<float>"})
    .SetInferShapeFn(PD_INFER_SHAPE(BevdetPostProcessInferShape))
    .SetInferDtypeFn(PD_INFER_DTYPE(PostProcessInferDtype));
