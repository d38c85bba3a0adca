// TEST INFRASTRUCTURE ONLY — not part of the product.
// extern "C" entry points around the UNMODIFIED reference CUDA launchers, compiled
// for sm_90a from where they lie in a Paddle3D checkout ($P3D_REFERENCE) by oracle/Makefile.  These
// are "the kernels to beat" and the GPU-side parity oracle (raw device pointers in/out):
//   paddle3d/ops/iou3d_nms/iou3d_nms_kernel.cu:436-482   BoxesOverlap/BoxesIouBev/Nms/NmsNormal launchers
//   paddle3d/ops/centerpoint_postprocess/iou3d_nms_kernel.cu:341-352  indexed NmsLauncher
//   paddle3d/ops/bev_pool_v2/bev_pool_cuda.cu:98-116      bev_pool_v2 / bev_pool_v2_grad
#include <cuda_runtime.h>
#include <stdint.h>

#if defined(P3D_REF_IOU3D)
void BoxesOverlapLauncher(const cudaStream_t &stream, const int num_a, const float *boxes_a, const int num_b,
                          const float *boxes_b, float *ans_overlap);
void BoxesIouBevLauncher(const cudaStream_t &stream, const int num_a, const float *boxes_a, const int num_b,
                         const float *boxes_b, float *ans_iou);
void NmsLauncher(const cudaStream_t &stream, const float *boxes, int64_t *mask, int boxes_num,
                 float nms_overlap_thresh);
void NmsNormalLauncher(const cudaStream_t &stream, const float *boxes, int64_t *mask, int boxes_num,
                       float nms_overlap_thresh);
#elif defined(P3D_REF_CPP)
void NmsLauncher(const cudaStream_t &stream, const float *bboxes, const int *index, const int64_t *sorted_index,
                 const int num_bboxes, const int num_bboxes_for_nms, const float nms_overlap_thresh,
                 const int decode_bboxes_dims, int64_t *mask);
#elif defined(P3D_REF_BEVPOOL)
void bev_pool_v2(int c, int n_intervals, const float *depth, const float *feat, const int *ranks_depth,
                 const int *ranks_feat, const int *ranks_bev, const int *interval_starts,
                 const int *interval_lengths, float *out);
void bev_pool_v2_grad(int c, int n_intervals, const float *out_grad, const float *depth, const float *feat,
                      const int *ranks_depth, const int *ranks_feat, const int *ranks_bev,
                      const int *interval_starts, const int *interval_lengths, float *depth_grad,
                      float *feat_grad);
#endif

extern "C" {
#if defined(P3D_REF_IOU3D)
void ref_boxes_overlap_gpu(void *stream, int na, const float *a, int nb, const float *b, float *out) {
  BoxesOverlapLauncher((cudaStream_t)stream, na, a, nb, b, out);
}
void ref_boxes_iou_bev_gpu(void *stream, int na, const float *a, int nb, const float *b, float *out) {
  BoxesIouBevLauncher((cudaStream_t)stream, na, a, nb, b, out);
}
void ref_nms_mask_gpu(void *stream, const float *boxes, int64_t *mask, int n, float thr) {
  NmsLauncher((cudaStream_t)stream, boxes, mask, n, thr);
}
void ref_nms_normal_mask_gpu(void *stream, const float *boxes, int64_t *mask, int n, float thr) {
  NmsNormalLauncher((cudaStream_t)stream, boxes, mask, n, thr);
}
#elif defined(P3D_REF_CPP)
void ref_cpp_nms_mask_gpu(void *stream, const float *bboxes, const int *index, const int64_t *sorted_index,
                          int num_bboxes, int num_for_nms, float thr, int dims, int64_t *mask) {
  NmsLauncher((cudaStream_t)stream, bboxes, index, sorted_index, num_bboxes, num_for_nms, thr, dims, mask);
}
#elif defined(P3D_REF_BEVPOOL)
// reference launches on the default stream (bev_pool_cuda.cu:102)
void ref_bev_pool_v2_gpu(int c, int n_intervals, const float *depth, const float *feat, const int *ranks_depth,
                         const int *ranks_feat, const int *ranks_bev, const int *interval_starts,
                         const int *interval_lengths, float *out) {
  bev_pool_v2(c, n_intervals, depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths,
              out);
}
void ref_bev_pool_v2_grad_gpu(int c, int n_intervals, const float *out_grad, const float *depth, const float *feat,
                              const int *ranks_depth, const int *ranks_feat, const int *ranks_bev,
                              const int *interval_starts, const int *interval_lengths, float *depth_grad,
                              float *feat_grad) {
  bev_pool_v2_grad(c, n_intervals, out_grad, depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_starts,
                   interval_lengths, depth_grad, feat_grad);
}
#endif
}
