/*
 * p3d_b200.h — C ABI of libp3d_b200.so: the H100 (sm_90a) implementation of Paddle3D's
 * point-cloud-to-BEV hot path.  This is the drop-in boundary: every entry point below is what a
 * Paddle custom-op kernel function (PD_BUILD_OP ... SetKernelFn) for this path binds to; the
 * reference interface each one replaces is cited as file:line under PaddlePaddle/Paddle3D @ 3259dabe.
 *
 * Conventions
 *   - plain pointers and sizes only; no C++/torch/paddle types.
 *   - unless a name ends in `_host`, every data pointer is a DEVICE pointer; attribute arrays
 *     (voxel_size, point_cloud_range, ...) are HOST pointers read before the launch.
 *   - `stream` is a cudaStream_t passed as void*.  Calls only enqueue work: they never allocate,
 *     never synchronise and never touch the default stream.  Data-dependent counts are written to
 *     device scalars; the caller reads them back when (and if) it needs them.
 *   - scratch memory is caller-provided: `p3d_<op>_workspace_bytes(...)` gives the size, any
 *     256-byte aligned device buffer of at least that size works, contents need not be preserved.
 *   - return value: 0 on success, negative p3d_status on failure (never throws).
 *     p3d_status_string() gives the message a PD_THROW would carry.
 */
#ifndef P3D_B200_H_
#define P3D_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void *p3d_stream_t; /* cudaStream_t */

enum p3d_status {
  P3D_OK = 0,
  P3D_ERR_INVALID_ARG = -1,   /* bad shape / null pointer / unsupported attribute */
  P3D_ERR_WORKSPACE = -2,     /* workspace_bytes smaller than p3d_*_workspace_bytes() */
  P3D_ERR_CUDA = -3,          /* a CUDA runtime call or launch failed (see p3d_last_cuda_error) */
  P3D_ERR_UNSUPPORTED = -4    /* valid in the reference but outside this build's limits */
};

const char *p3d_status_string(int status);
int p3d_last_cuda_error(void); /* cudaError_t of the last P3D_ERR_CUDA on this thread */
int p3d_abi_version(void);

/* ---------------------------------------------------------------------------------------------
 * hard_voxelize      replaces paddle3d/ops/voxel/voxelize_op.cc:149-166 (op `hard_voxelize`,
 *                    registration :183-191; CUDA path voxelize_op.cu:208-346).
 * Semantics are those of the reference CPU kernel (voxelize_op.cc:19-82), deterministically:
 * voxels numbered in first-appearance order of their first point, capped at max_voxels; each voxel
 * keeps its first max_points points in input order.
 *   points               [num_points, num_point_dim] fp32 (num_point_dim >= 3)
 *   voxel_size_host[3], point_cloud_range_host[6]     attrs
 *   voxels               [max_voxels, max_points, num_point_dim] fp32, fully written (zero padded)
 *   coords               [max_voxels, 3] int32 (z, y, x), zero beyond num_voxels
 *   num_points_per_voxel [max_voxels] int32, zero beyond num_voxels
 *   num_voxels           [1] int32
 * ------------------------------------------------------------------------------------------- */
size_t p3d_hard_voxelize_workspace_bytes(int64_t num_points, int max_points, int max_voxels);
int p3d_hard_voxelize(const float *points, int64_t num_points, int num_point_dim, const float *voxel_size_host,
                      const float *point_cloud_range_host, int max_points, int max_voxels, float *voxels,
                      int32_t *coords, int32_t *num_points_per_voxel, int32_t *num_voxels, void *workspace,
                      size_t workspace_bytes, p3d_stream_t stream);

/* Fused front end used by the CenterPoint pipeline: hard_voxelize + VoxelMean
 * (paddle3d/models/voxel_encoders/voxel_encoder.py:49-57) + HardVoxelizer's batch-id pad
 * (paddle3d/models/voxelizers/voxelize.py:39-58) without materialising the padded voxels tensor.
 *   mean   [max_voxels, num_point_dim] fp32 (rows >= num_voxels zero)
 *   coors4 [max_voxels, 4] int32 (batch_id, z, y, x)  */
int p3d_voxelize_mean(const float *points, int64_t num_points, int num_point_dim, const float *voxel_size_host,
                      const float *point_cloud_range_host, int max_points, int max_voxels, int batch_id,
                      float *mean, int32_t *coors4, int32_t *num_points_per_voxel, int32_t *num_voxels,
                      void *workspace, size_t workspace_bytes, p3d_stream_t stream);

/* VoxelMean alone: voxels [num_voxels_cap, max_points, F] -> mean [num_voxels_cap, F]; rows whose
 * index >= *num_voxels_dev (device scalar, may be NULL = all rows) are written as zero. */
int p3d_voxel_mean(const float *voxels, const int32_t *num_points_per_voxel, const int32_t *num_voxels_dev,
                   int num_voxels_cap, int max_points, int num_point_dim, float *mean, p3d_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * pillar_scatter / sparse to_dense     replaces PointPillarsScatter.forward_batch
 *   (paddle3d/models/middle_encoders/pillar_scatter.py:57-105: zeros + paddle.scatter + transpose)
 *   and SparseResNet3D's to_dense + transpose + reshape (sparse_resnet.py:202-206).
 *   feats  [n, C] fp32;  coords [n, 4] int32 (batch, z, y, x);  n_dev: device count (NULL = n_cap)
 *   out    [batch, C, D, ny, nx] fp32 fully written; a pillar canvas is the D == 1 case and uses
 *          index y*nx + x (z ignored), later rows win on duplicate cells.
 * ------------------------------------------------------------------------------------------- */
size_t p3d_scatter_dense_workspace_bytes(int batch, int D, int ny, int nx);
int p3d_scatter_dense(const float *feats, const int32_t *coords, const int32_t *n_dev, int n_cap, int C,
                      int batch, int D, int ny, int nx, int use_z, float *out, void *workspace,
                      size_t workspace_bytes, p3d_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * bev_pool_v2 / bev_pool_v2_bkwd      replace paddle3d/ops/bev_pool_v2/bev_pool.cc:30-54, :56-96
 *   (registrations :111-118 and ops/bev_pool_v2_backward/bev_pool_bkwd.cc:75-80; kernels
 *   bev_pool_cuda.cu:18-96).  NOTE the reference argument order: lengths before starts.
 *   depth [B*N, D, H, W] fp32 (flat-indexed by ranks_depth); feat [B*N, H, W, C] fp32;
 *   ranks_* [n_points] int32; interval_* [n_intervals] int32; out [out_numel] fp32 zero-filled here.
 * ------------------------------------------------------------------------------------------- */
int p3d_bev_pool_v2(const float *depth, const float *feat, const int32_t *ranks_depth, const int32_t *ranks_feat,
                    const int32_t *ranks_bev, const int32_t *interval_lengths, const int32_t *interval_starts,
                    int n_intervals, int c, float *out, int64_t out_numel, p3d_stream_t stream);
int p3d_bev_pool_v2_bkwd(const float *out_grad, const float *depth, const float *feat, const int32_t *ranks_depth,
                         const int32_t *ranks_feat, const int32_t *ranks_bev, const int32_t *interval_lengths,
                         const int32_t *interval_starts, int n_intervals, int c, float *depth_grad,
                         int64_t depth_numel, float *feat_grad, int64_t feat_numel, p3d_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * iou3d_nms      replaces paddle3d/ops/iou3d_nms/iou3d_nms.cpp:44-204 (registrations
 *                iou3d_nms_api.cpp:73-108).  boxes are [n, 7] = x, y, z, dx, dy, dz, heading.
 * ------------------------------------------------------------------------------------------- */
int p3d_boxes_overlap_bev(const float *boxes_a, int num_a, const float *boxes_b, int num_b, float *overlap,
                          p3d_stream_t stream);
int p3d_boxes_iou_bev(const float *boxes_a, int num_a, const float *boxes_b, int num_b, float *iou,
                      p3d_stream_t stream);
/* nms_gpu / nms_normal_gpu: boxes already sorted by score.  keep [n] int32 (first *num_keep valid),
 * num_keep [1] int32 — both on the DEVICE (the reference finishes on the host; here the greedy
 * reduction runs on the GPU with no sync).  normal != 0 selects the axis-aligned IoU. */
size_t p3d_nms_workspace_bytes(int n);
int p3d_nms(const float *boxes, int n, float nms_overlap_thresh, int normal, int32_t *keep, int32_t *num_keep,
            void *workspace, size_t workspace_bytes, p3d_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * centerpoint_postprocess      replaces paddle3d/ops/centerpoint_postprocess/postprocess.cc:34-104
 *                              (postprocess_gpu, postprocess.cu:104-280), batch size 1.
 *   hm/reg/height/dim/vel/rot: HOST arrays of T device pointers to the per-task NCHW tensors
 *   hm_channels_host[T]; attrs as in the op.  num_classes_host[T] are the label offsets.
 *   Outputs (device), sized for the worst case rows_cap = T * max(nms_post_max_size, 1):
 *     bboxes [rows_cap, 9 or 7], scores [rows_cap], labels [rows_cap] int64,
 *     counts [T + 1] int32: rows per task, then the total number of valid rows.
 *   Score-sort tie order is defined as ascending cell index.
 * ------------------------------------------------------------------------------------------- */
size_t p3d_centerpoint_postprocess_workspace_bytes(int num_tasks, int feat_h, int feat_w, int nms_pre_max_size,
                                                    int nms_post_max_size);
int p3d_centerpoint_postprocess(int num_tasks, const float *const *hm, const int32_t *hm_channels_host,
                                const float *const *reg, const float *const *height, const float *const *dim,
                                const float *const *vel, const float *const *rot, int feat_h, int feat_w,
                                const float *voxel_size_host, const float *point_cloud_range_host,
                                const float *post_center_range_host, const int32_t *num_classes_host,
                                int down_ratio, float score_threshold, float nms_iou_threshold,
                                int nms_pre_max_size, int nms_post_max_size, int with_velocity, float *bboxes,
                                float *scores, int64_t *labels, int32_t *counts, void *workspace,
                                size_t workspace_bytes, p3d_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * bevdet_postprocess      BEVDet's own box decode, CenterHead.get_bboxes (CenterPointBBoxCoder.decode,
 *                         get_task_detections with scale-NMS, circle_nms), batch size 1.  PARITY UNPINNED: the rules
 *                         below are recalled from BEVDet's head, not checked against a checkout of it.
 *   hm/reg/height/dim/vel/rot, hm_channels_host[T]: as centerpoint_postprocess.  Per task t with C_t classes:
 *   1. every (class c, cell i) with score = sigmoid(hm[c, i]) > score_threshold is a candidate (not the cell's arg-max);
 *   2. the max_num best of them, by descending score; equal scores order by ascending c * H*W + i (torch.topk leaves
 *      ties undefined; this is the order defined here);
 *   3. x = (xs + reg0) * out_size_factor * voxel_size[0] + point_cloud_range[0], y likewise, z = height,
 *      dims = exp(dim), rot = atan2f(rot0, rot1), velocity copied (fp32, each operation rounded on its own);
 *   4. kept iff the DECODED (x, y, z) lies in post_center_range, both ends inclusive;
 *   5. suppression over the first pre_max_size survivors in score order; a box is suppressed by a kept box ahead of it
 *      nms_type_host[t] == P3D_BEVDET_NMS_ROTATE: when the rotated BEV IoU of (x, y, z, dx*f, dy*f, dz, rot) exceeds
 *        nms_thr_host[t], f = rescale_host[class] (one factor per class, the tasks' classes concatenated; no w/l swap);
 *      nms_type_host[t] == P3D_BEVDET_NMS_CIRCLE: when the squared centre distance (fp32) is <= min_radius_host[t];
 *      the first post_max_size kept boxes survive;
 *   6. rows are (x, y, z - dz/2, dx, dy, dz, rot, vx, vy): bottom centre, dims unscaled (the reference multiplies by f
 *      and divides again: at most one ulp from the value written here), label = c + label_offset_host[t].
 *   Outputs (device), sized for the worst case: bboxes [T * post_max_size, 9], scores, labels int64,
 *   counts [T + 1] int32: rows per task, then the total.  An empty task contributes no row.
 *   Non-finite inputs: a NaN logit is no candidate and +inf scores 1, so every score is finite; a candidate whose
 *   decoded centre is NaN or infinite fails the range test, and one whose dims, rot or velocity are NaN or infinite
 *   is dropped with it (the reference has no such rule: it would carry the value into its NMS).  Every row is finite.
 *   Limits (P3D_ERR_UNSUPPORTED): T <= 16, at most 64 classes over all tasks, max_num <= 393216.
 * ------------------------------------------------------------------------------------------- */
#define P3D_BEVDET_NMS_ROTATE 0
#define P3D_BEVDET_NMS_CIRCLE 1
size_t p3d_bevdet_postprocess_workspace_bytes(int num_tasks, const int32_t *hm_channels_host, int feat_h, int feat_w,
                                              int max_num);
int p3d_bevdet_postprocess(int num_tasks, const float *const *hm, const int32_t *hm_channels_host,
                           const float *const *reg, const float *const *height, const float *const *dim,
                           const float *const *vel, const float *const *rot, int feat_h, int feat_w,
                           const float *voxel_size_host, const float *point_cloud_range_host,
                           const float *post_center_range_host, int out_size_factor, float score_threshold,
                           int max_num, int pre_max_size, int post_max_size, const int32_t *nms_type_host,
                           const float *nms_thr_host, const float *min_radius_host, const float *rescale_host,
                           const int32_t *label_offset_host, float *bboxes, float *scores, int64_t *labels,
                           int32_t *counts, void *workspace, size_t workspace_bytes, p3d_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Sparse 3-D convolution     replaces the paddle.sparse.nn layer calls made by SparseResNet3D /
 *   SparseNet3D (paddle3d/models/middle_encoders/sparse_resnet.py:31-60,84-111,125-206;
 *   sparsenet.py:38-52,75-155): SubmConv3D / Conv3D (+ BatchNorm(eval) + residual add + ReLU fused).
 *
 * Rulebook ("neighbour map") build.  coords are [n, 4] int32 (batch, z, y, x); spatial = (D, H, W).
 *   p3d_sparse_rulebook_subm : nbr [n_cap, K] int32, nbr[i][k] = input row at coord(i) - pad + k or -1
 *                              (K = kD*kH*kW, pad = k/2; shared by every SubM layer of a stage).
 *   p3d_sparse_rulebook_conv : strided Conv3D: writes the output coordinate list out_coords
 *                              [out_cap, 4], the device counters n_out_dev (int32[4]) and
 *                              nbr [out_cap, K] with nbr[o][k] = input row at o*stride - pad + k or -1.
 *   Output site order: first appearance.  Walk the input rows in row order and, within a row, the
 *   taps k = (kz*kH + ky)*kW + kx in order; a site is appended the first time it is generated
 *   (output o from input c under tap k when c = o*stride - pad + k).  The order depends only on
 *   the input index set: the same in every run, on every stream, eager or captured, and from both
 *   strided entry points.  Malformed input: of rows sharing a coordinate the LAST stands for it
 *   (it is the row nbr names) and the others generate no sites; rows outside the input grid
 *   (batch or spatial) generate no sites and are in no map.  When out_cap is too small the rows
 *   kept are the first out_cap sites of this order (while the output table, sized for 2*out_cap
 *   rows, holds every site: n_out_dev[3] = 0).
 *   n_in_dev / n_out_dev are device scalars so the whole backbone runs without a host sync.
 *   n_out_dev[0] = number of output sites (clamped to out_cap), n_out_dev[1] = 1 if sites were
 *   dropped because out_cap was too small, n_out_dev[2] = unclamped count (a lower bound once the
 *   output table itself is full), n_out_dev[3] = internal table-full flag.
 * ------------------------------------------------------------------------------------------- */
size_t p3d_sparse_rulebook_workspace_bytes(int64_t n_in_cap, int64_t n_out_cap);
int p3d_sparse_rulebook_subm(const int32_t *coords, const int32_t *n_in_dev, int64_t n_in_cap, int batch,
                             const int *spatial_host, const int *ksize_host, int32_t *nbr, void *workspace,
                             size_t workspace_bytes, p3d_stream_t stream);
int p3d_sparse_rulebook_conv(const int32_t *coords, const int32_t *n_in_dev, int64_t n_in_cap, int batch,
                             const int *spatial_host, const int *ksize_host, const int *stride_host,
                             const int *pad_host, int32_t *out_coords, int32_t *n_out_dev, int64_t out_cap,
                             int32_t *nbr, void *workspace, size_t workspace_bytes, p3d_stream_t stream);

/* Caller-owned coordinate tables (one per index set / resolution level): the same rulebooks with every level's
 * table built exactly once per frame (the two calls above run this path on tables carved out of their workspace).
 * p3d_sparse_table_build hashes an index set's coordinates; p3d_sparse_rulebook_subm_t only looks neighbours up in it.
 * Tables are p3d_sparse_table_bytes(rows_cap) bytes, 16-byte aligned; the size includes the scratch a strided level
 * numbering its sites into the table uses. */
size_t p3d_sparse_table_bytes(int64_t rows_cap);
int p3d_sparse_table_build(const int32_t *coords, const int32_t *n_dev, int64_t n_cap, int batch,
                           const int *spatial_host, void *table, size_t table_bytes, p3d_stream_t stream);
int p3d_sparse_rulebook_subm_t(const int32_t *coords, const int32_t *n_dev, int64_t n_cap, int batch,
                               const int *spatial_host, const int *ksize_host, const void *table, size_t table_bytes,
                               int32_t *nbr, p3d_stream_t stream);

/* One resolution level in two launches: the strided conv of p3d_sparse_rulebook_conv (out_coords, n_out_dev, nbr) with
 * the inputs looked up in table_in; table_out is left holding the table of the OUTPUT index set (a by-product of
 * enumerating its sites), ready for the next stage.  When nbr_subm is given, also the SubM neighbour map
 * [out_cap, prod(subm_ksize)] of the NEW level (odd kernel, "same" padding) looked up in table_out - what a following
 * p3d_sparse_rulebook_subm_t on the output index set would return. */
int p3d_sparse_rulebook_level_t(const int32_t *coords, const int32_t *n_in_dev, int64_t n_in_cap, int batch,
                                const int *spatial_host, const int *ksize_host, const int *stride_host,
                                const int *pad_host, const void *table_in, size_t table_in_bytes, int32_t *out_coords,
                                int32_t *n_out_dev, int64_t out_cap, void *table_out, size_t table_out_bytes,
                                int32_t *nbr, const int *subm_ksize_host, int32_t *nbr_subm, p3d_stream_t stream);

/* Unfused elementwise epilogue (BatchNorm(eval) / sparse.add / ReLU on a materialised tensor):
 *   out[r, c] = act(x[r, c] * scale[c] + shift[c] (+ residual[r, c])); out may alias x. */
int p3d_sparse_affine_act(const float *x, const int32_t *n_dev, int64_t n_cap, int C, const float *scale,
                          const float *shift, const float *residual, int relu, float *out, p3d_stream_t stream);

/* Gather-GEMM-scatter in output-stationary form:
 *   out[o, :] = act( (sum_k in[nbr[o][k], :] @ W[k]) * scale + shift (+ residual[o, :]) )
 *   in [n_in, Cin] fp32; W [K, Cin, Cout] fp32 (Paddle's [kD,kH,kW,Cin,Cout]); scale/shift [Cout]
 *   (BatchNorm(eval) and conv bias folded by the caller; NULL = identity); residual [n_out, Cout] or
 *   NULL; relu != 0 applies max(.,0).  n_out_dev: device row count (NULL = n_out_cap rows).
 *   precision: P3D_CONV_FP32 = fp32 FMA on CUDA cores; P3D_CONV_TF32X3 = wgmma tensor cores with
 *   3xTF32 split accumulation in registers (fp32-level accuracy). */
enum p3d_conv_precision { P3D_CONV_FP32 = 0, P3D_CONV_TF32X3 = 1 };
/* Weight pre-pack for P3D_CONV_TF32X3 (once per layer): splits W [K, Cin, Cout] into tf32 hi / lo and lays it out
 * as the shared-memory image the tensor-core kernel streams with cp.async.bulk.  Needs Cin, Cout multiples of
 * 16 (Cin multiple of 32 above 32); returns P3D_ERR_UNSUPPORTED otherwise (use P3D_CONV_FP32 for such layers).
 * With precision == P3D_CONV_TF32X3 the `weight` argument of p3d_sparse_conv_gather_gemm is this packed buffer. */
size_t p3d_sparse_conv_packed_weight_bytes(int K, int Cin, int Cout);
int p3d_sparse_conv_pack_weights(const float *weight, int K, int Cin, int Cout, float *packed, p3d_stream_t stream);
int p3d_sparse_conv_gather_gemm(const float *in, const int32_t *nbr, const int32_t *n_out_dev, int64_t n_out_cap,
                                int K, int Cin, int Cout, const float *weight, const float *scale,
                                const float *shift, const float *residual, int relu, int precision, float *out,
                                p3d_stream_t stream);

/* Tensor-core gather-GEMM with split-K over the kernel taps for the wide layers (Cout >= 64): layers with few
 * 128-row tiles are spread over 2 CTAs per tile; partial sums go to the caller's scratch slabs and are added in a
 * fixed order by a finalize pass that also applies the epilogue (deterministic).  Same contract as
 * p3d_sparse_conv_gather_gemm(precision = P3D_CONV_TF32X3); with workspace == NULL it runs unsplit. */
size_t p3d_sparse_conv_splitk_workspace_bytes(int64_t n_out_cap, int Cin, int Cout);
int p3d_sparse_conv_gather_gemm_tf32x3_ws(const float *in, const int32_t *nbr, const int32_t *n_out_dev,
                                          int64_t n_out_cap, int K, int Cin, int Cout, const float *packed_weight,
                                          const float *scale, const float *shift, const float *residual, int relu,
                                          float *out, void *workspace, size_t workspace_bytes, p3d_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Split-row activations for the tensor-core path.  A "split" row tensor stores every row as its tf32 hi half
 * followed by its tf32 lo half: [n][2][C] fp32 words (x ~= hi + lo, error <= 2^-22 |x|).  Keeping activations in
 * this form between sparse-conv layers moves the 3xTF32 split out of the gather loop (paid once per produced
 * element instead of once per gathering neighbour) and lets the kernel gather with cp.async.  Both row layouts run on
 * the same tensor-core kernel (csrc/sparse_conv_tc.cu) with the same arithmetic.
 *   p3d_rows_convert_layout: src_layout 0 = fp32 rows [n, C] -> split; 1 = split -> fp32 rows (hi + lo).
 *   p3d_sparse_conv_gather_gemm_split: same contract as p3d_sparse_conv_gather_gemm(precision = TF32X3) with
 *     in_split [n_in][2][Cin], residual_split [n_out][2][Cout] or NULL, packed weights
 *     (p3d_sparse_conv_pack_weights), and out_f32 [n_out, Cout] and / or out_split [n_out][2][Cout] (either may be
 *     NULL, not both) and a 16-byte aligned nbr.  Persistent grid sized to the device row count.
 *   p3d_sparse_conv_gather_gemm_split_ws: the same with a scratch buffer of
 *     p3d_sparse_conv_splitk_workspace_bytes(n_out_cap, Cin, Cout) bytes; when present the wide layers run split-K over
 *     taps (partial sums in the scratch slabs, added in slab order by a finalize kernel: deterministic).
 * ------------------------------------------------------------------------------------------- */
int p3d_rows_convert_layout(const float *src, int src_layout, const int32_t *n_dev, int64_t n_cap, int C, float *dst,
                            p3d_stream_t stream);
int p3d_sparse_conv_gather_gemm_split(const float *in_split, const int32_t *nbr, const int32_t *n_out_dev,
                                      int64_t n_out_cap, int K, int Cin, int Cout, const float *packed_weight,
                                      const float *scale, const float *shift, const float *residual_split, int relu,
                                      float *out_f32, float *out_split, p3d_stream_t stream);
int p3d_sparse_conv_gather_gemm_split_ws(const float *in_split, const int32_t *nbr, const int32_t *n_out_dev,
                                         int64_t n_out_cap, int K, int Cin, int Cout, const float *packed_weight,
                                         const float *scale, const float *shift, const float *residual_split, int relu,
                                         float *out_f32, float *out_split, void *workspace, size_t workspace_bytes,
                                         p3d_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * fp16-pair ("H16") activations: the default tensor-core path of the sparse layers (csrc/sparse_conv_f16.cu).
 * x = hi + lo' * 2^-11 with hi = fp16(x), lo' = fp16((x - hi) * 2^11): the same 22 significant bits as the tf32 pair
 * in half the bytes (a row of C channels is 4*C bytes: groups of KC = min(C, 32) channels, each [hi KC | lo' KC] halfs).
 * Valid for |x| < 65504; values outside are saturated and bit 0 of *status_dev is set (use the tf32 split path for
 * such data).  Same layer contract as p3d_sparse_conv_gather_gemm_split (paddle.sparse.nn.SubmConv3D / Conv3D +
 * BatchNorm(eval) + add + ReLU, sparse_resnet.py:31-60,84-111):
 *   p3d_sparse_conv_f16_pack_weights   W[K][Cin][Cout] fp32 -> k-blocks of the (hi | lo') weight image
 *   p3d_rows_convert_h16               to_h16 != 0: fp32 rows [n, C] -> H16 rows; 0: H16 rows -> fp32 rows
 *   p3d_sparse_conv_f16                persistent kernel, split-K over taps chosen on the device (up to max_splits,
 *                                      bounded by the workspace); workspace = p3d_sparse_conv_f16_workspace_bytes(...)
 *                                      bytes whose first align_up(tiles * 4) bytes (tickets) must be ZERO on first use
 *                                      (the kernel leaves them zero); workspace NULL or max_splits <= 1: no split.
 * ------------------------------------------------------------------------------------------- */
/* fp16-pair plumbing around the tensor-core layers: the 5-channel input layer emitting pair rows directly, and the last
 * level's rows scattered straight into the pixel H16 image [batch, ny, nx][D * C] the dense RPN reads (the fp16-pair form
 * of to_dense + transpose + reshape, sparse_resnet.py:202-206; duplicates impossible: sites are unique). */
int p3d_sparse_conv_small_cin_h16(const float *in, const int32_t *nbr, const int32_t *n_out_dev, int64_t n_out_cap, int K,
                                  int Cin, int Cout, const float *weight, const float *scale, const float *shift, int relu,
                                  float *out_f32, void *out_h16, int32_t *status_dev, p3d_stream_t stream);
int p3d_sparse_rows_to_pixel_h16(const void *rows_h16, const int32_t *coords, const int32_t *n_dev, int n_cap, int C,
                                 int batch, int D, int ny, int nx, void *out_pixel_h16, p3d_stream_t stream);
size_t p3d_sparse_conv_f16_packed_weight_bytes(int K, int Cin, int Cout);
int p3d_sparse_conv_f16_pack_weights(const float *weight, int K, int Cin, int Cout, void *packed, int32_t *status_dev,
                                     p3d_stream_t stream);
int p3d_rows_convert_h16(const void *src, int to_h16, const int32_t *n_dev, int64_t n_cap, int C, void *dst,
                         int32_t *status_dev, p3d_stream_t stream);
size_t p3d_sparse_conv_f16_workspace_bytes(int64_t n_out_cap, int Cout, int max_splits);
int p3d_sparse_conv_f16(const void *in_h16, const int32_t *nbr, const int32_t *n_out_dev, int64_t n_out_cap, int K,
                        int Cin, int Cout, const void *packed_weight, const float *scale, const float *shift,
                        const void *residual_h16, int relu, float *out_f32, void *out_h16, void *workspace,
                        size_t workspace_bytes, int max_splits, int32_t *status_dev, p3d_stream_t stream);

/* Narrow layers (Cin, Cout) in {(16,16), (16,32), (32,32)}: register gather + warp MMA (csrc/sparse_conv_wm.cu), same
 * H16 rows in and out, same fused epilogue and the same three-product arithmetic as p3d_sparse_conv_f16; only the weight
 * image differs (mma.sync fragment order, k permuted so that a lane's fragment is 4 contiguous channels of a row).
 * Missing neighbours cost nothing here (predicated-off loads), unlike the staged gathers of the wgmma kernel.
 * Work is cut stream-K style into equal (tile, tap) ranges per warp; a tile cut by a range boundary is summed by the last
 * warp to finish it, pieces in warp order (deterministic).  workspace = p3d_sparse_conv_wm_workspace_bytes(...) bytes whose
 * first align_up(ceil(n_out_cap / 16) * 4) bytes (tickets) must be ZERO on first use (the kernel leaves them zero).
 * p3d_sparse_conv_wm_packed_weight_bytes returns 0 for unsupported shapes. */
size_t p3d_sparse_conv_wm_packed_weight_bytes(int K, int Cin, int Cout);
int p3d_sparse_conv_wm_pack_weights(const float *weight, int K, int Cin, int Cout, void *packed, int32_t *status_dev,
                                    p3d_stream_t stream);
size_t p3d_sparse_conv_wm_workspace_bytes(int64_t n_out_cap, int Cout);
int p3d_sparse_conv_wm(const void *in_h16, const int32_t *nbr, const int32_t *n_out_dev, int64_t n_out_cap, int K, int Cin,
                       int Cout, const void *packed_weight, const float *scale, const float *shift,
                       const void *residual_h16, int relu, float *out_f32, void *out_h16, void *workspace,
                       size_t workspace_bytes, int32_t *status_dev, p3d_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * SURVEY.md 8f-1: dense 2-D convolution on wgmma (tf32 pairs) for the RPN / neck /
 * CenterHead (reference: backbones/second_backbone.py:72-120, necks/second_fpn.py:99-160,
 * detection/centerpoint/center_head.py:43-220).  Images are "pixel split rows" [B*H*W][2][C] (the split-row format
 * of the sparse layers with row = pixel).
 *   p3d_nchw_to_pixel_split: fp32 [B, C, H, W] -> pixel split rows.
 *   p3d_dense_conv2d_packed_weight_bytes / p3d_dense_conv2d_split: weights = per N tile (n_tile = 16 | 64 | 128 output
 *     channels, zero-padded) the image p3d_sparse_conv_pack_weights makes of W[tap][Cin][n_tile], tiles concatenated.
 *     up == 1: Conv2D(kh x kw, stride 1 | 2, zero padding pad); up > 1: Conv2DTranspose with kernel = stride = up
 *     (pass kh = kw = stride = up, pad = 0).  Epilogue v * scale[c] + shift[c] (either may be NULL), optional ReLU.
 *     Output: split rows of out_C channels written at column out_c0 (channel concat), and / or fp32 NCHW planes
 *     [B, Cout, out_H, out_W].  Cin % 32 == 0; Cout % 16 == 0 for split-row output.
 * ------------------------------------------------------------------------------------------- */
int p3d_nchw_to_pixel_split(const float *in, int B, int C, int H, int W, float *out_split, p3d_stream_t stream);
size_t p3d_dense_conv2d_packed_weight_bytes(int taps, int Cin, int Cout, int n_tile);
int p3d_dense_conv2d_split(const float *in_split, int B, int H, int W, int Cin, const float *packed_weight, int Cout,
                           int n_tile, int kh, int kw, int stride, int pad, int up, const float *scale,
                           const float *shift, int relu, float *out_split, int out_C, int out_c0, float *out_nchw,
                           p3d_stream_t stream);

/* The grouped 3x3 output convs of CenterHead's SeparateHeads (center_head.py:80-117) as one CUDA-core launch.  in_split: pixel split rows [B*H*W][2][in_C]; group g convolves
 * channels [g*Cin, (g+1)*Cin) with weight [groups][9][Cin][4] (outputs zero-padded to 4) + bias [groups][4] and
 * writes cnt[g] fp32 planes from plane0[g] of out_nchw [B, planes, H, W] (plane0 / cnt are HOST arrays). */
int p3d_head_final_conv(const float *in_split, int B, int H, int W, int in_C, int Cin, int groups, const float *weight,
                        const float *bias, const int32_t *plane0_host, const int32_t *cnt_host, int planes,
                        float *out_nchw, p3d_stream_t stream);

/* fp16-pair dense convolution (csrc/dense_conv_f16.cu): same layer contract as p3d_dense_conv2d_split on pixel H16
 * rows [B*H*W][C / 32 groups][hi 32 | lo' 32] halfs.  3x3 / stride 1 / pad 1 layers load the haloed tile once per
 * 32-channel group and read the 9 taps through shifted wgmma descriptors; everything else loads one box per tap.
 * mode 0 = auto, 1 = force per-tap loads (other values: P3D_ERR_INVALID_ARG); m_tiles 0 = auto, 1 or 2 M tiles
 * (8 x 16 pixels each) per work item; n_tile 64 or 128. */
int p3d_nchw_to_pixel_h16(const float *in, int B, int C, int H, int W, void *out_h16, int32_t *status_dev,
                          p3d_stream_t stream);
int p3d_pixel_h16_to_nchw(const void *in_h16, int B, int C, int H, int W, float *out, p3d_stream_t stream);
size_t p3d_dense_conv2d_f16_packed_weight_bytes(int taps, int Cin, int Cout, int n_tile);
int p3d_dense_conv2d_f16_pack_weights(const float *weight_tci, int taps, int Cin, int n_tile, void *packed,
                                      int32_t *status_dev, p3d_stream_t stream);
/* ---------------------------------------------------------------------------------------------
 * bev_pool rank preparation      replaces LSSViewTransformer.voxel_pooling_prepare_v2
 *   (paddle3d/models/transformers/bevdet_transformer.py:230-274): frustum points coor [B, N, D, H, W, 3] fp32 ->
 *   ranks_bev / ranks_depth / ranks_feat sorted by ranks_bev (ties: ascending point index = stable argsort),
 *   interval_starts / interval_lengths; all outputs int32 [B*N*D*H*W] (capacity), counts_dev = {n_kept, n_intervals}.
 *   Entries beyond the counts are zero, except interval_starts (left unwritten).  grid_size_host = (X, Y, Z) cells,
 *   lower bound / interval per axis (x, y, z).  B * X * Y * Z <= 2^31, so that every rank (at most cells - 1) is an
 *   int32, and B * N * D * H * W <= 2^31 - 1 (P3D_ERR_UNSUPPORTED otherwise).
 * ------------------------------------------------------------------------------------------- */
size_t p3d_bev_pool_prepare_workspace_bytes(int64_t num_points);
int p3d_bev_pool_prepare(const float *coor, int B, int N, int D, int H, int W, const float *grid_lower_bound_host,
                         const float *grid_interval_host, const int32_t *grid_size_host, int32_t *ranks_bev,
                         int32_t *ranks_depth, int32_t *ranks_feat, int32_t *interval_starts, int32_t *interval_lengths,
                         int32_t *counts_dev, void *workspace, size_t workspace_bytes, p3d_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * LSS view transform (LSSViewTransformer, bevdet_transformer.py:147-316, PARITY UNPINNED: no checkout was read; the
 * restatement follows BEVDet's get_lidar_coor(sensor2ego, ego2global, cam2imgs, post_rots, post_trans, bda) with a 3x3
 * bda).  One camera descriptor per (b, n), row-major, computed on the host in fp64 and rounded to fp32 once.
 * ------------------------------------------------------------------------------------------- */
typedef struct p3d_lss_camera {
  float inv_post_rot[9]; /* inv(post_rots) */
  float post_trans[3];
  float combine[9];      /* sensor2ego[:3, :3] . inv(cam2imgs) */
  float trans[3];        /* sensor2ego[:3, 3] */
} p3d_lss_camera;

/* get_lidar_coor fused with voxel_pooling_prepare_v2: the outputs, their capacity B*N*D*H*W, the tie order and the
 * workspace (p3d_bev_pool_prepare_workspace_bytes(B*N*D*H*W)) and the size limits (B*X*Y*Z <= 2^31) are those of
 * p3d_bev_pool_prepare, but the frustum points are computed in registers instead of read from a coor tensor.  cams [B*N] and bda [B, 9] are device buffers (refresh
 * them with a copy before each launch and one captured graph serves every calibration); axis_depth [D], axis_x [W],
 * axis_y [H] fp32 are create_frustum's arange(*depth), linspace(0, W_in - 1, W), linspace(0, H_in - 1, H).
 * coor (nullable): the ego points as [B, N, D, H, W, 3] fp32, what get_lidar_coor returns. */
int p3d_lss_prepare(const p3d_lss_camera *cams, const float *bda, const float *axis_depth, const float *axis_x,
                    const float *axis_y, int B, int N, int D, int H, int W, const float *grid_lower_bound_host,
                    const float *grid_interval_host, const int32_t *grid_size_host, float *coor, int32_t *ranks_bev,
                    int32_t *ranks_depth, int32_t *ranks_feat, int32_t *interval_starts, int32_t *interval_lengths,
                    int32_t *counts_dev, void *workspace, size_t workspace_bytes, p3d_stream_t stream);
/* Depth softmax + feature permute of view_transform, one launch: logits [BN, D, H, W] -> depth [BN, D, H, W] =
 * softmax over D (max subtracted, expf, sum in ascending d, one division); tran_feat [BN, C, H, W] -> feat [BN, H, W, C].
 * D <= 382 and C <= 370 (P3D_ERR_UNSUPPORTED above). */
int p3d_lss_depth_feat(const float *logits, const float *tran_feat, int BN, int D, int H, int W, int C, float *depth,
                       float *feat, p3d_stream_t stream);
/* p3d_lss_depth_feat from the depth net's pixel H16 rows rows_h16 [BN, H, W, in_C] (channels [0, D) the logits, [D, D + C)
 * the features; each value merged as hi + lo' 2^-11): writes what p3d_lss_depth_feat writes for those merged values,
 * bit for bit (same softmax operations in the same order).  in_C % 32 == 0, D + C <= in_C, rows_h16 16-byte aligned
 * (P3D_ERR_INVALID_ARG otherwise); D <= 370, BN <= 65535, BN * H * W * 4 * in_C bytes < 2^31 (P3D_ERR_UNSUPPORTED above). */
int p3d_lss_depth_feat_h16(const void *rows_h16, int BN, int H, int W, int in_C, int D, int C, float *depth, float *feat,
                           p3d_stream_t stream);
/* bev_pool_v2 with the interval count on the device (counts_dev[1], as p3d_bev_pool_prepare / p3d_lss_prepare write it;
 * capacity = length of the rank arrays), so that it can be captured once for every calibration.  Bit-identical to
 * p3d_bev_pool_v2 (same kernel).  out is zero-filled here: planar 0 -> [B, Z, Y, X, c], planar 1 -> [B, Z * c, Y, X]
 * with channel z * c + ch (view_transform's collapse_z layout).  c % 4 == 0, c <= 256, feat / out 16-byte aligned,
 * B * Z * Y * X <= 2^31 (the int32 ranks' range) (P3D_ERR_UNSUPPORTED otherwise). */
int p3d_bev_pool_v2_dev(const float *depth, const float *feat, const int32_t *ranks_depth, const int32_t *ranks_feat,
                        const int32_t *ranks_bev, const int32_t *interval_lengths, const int32_t *interval_starts,
                        const int32_t *counts_dev, int64_t capacity, int c, int B, int Z, int Y, int X, int planar,
                        float *out, p3d_stream_t stream);

/* Grouped 3x3 output convs of the CenterHead (center_head.py:80-117) as one tensor-core launch with the 9 taps in the
 * GEMM's N dimension (<= 3 output channels per group; a wider conv is split into several groups over the same input
 * slice): one [256 haloed pixels x Cin] x [Cin x 27] GEMM per 14 x 14 output tile, then every pixel adds its 9 shifted
 * partial sums.  Group g reads input channels [cin0[g], cin0[g] + Cin) of the in_C-channel H16 image (cin0_dev null:
 * g * Cin) and writes cnt[g] fp32 planes from plane0[g] (device int32 arrays); packed_weight: per group
 * p3d_dense_conv2d_f16_pack_weights(taps 1, Cin, n_tile 32) of W2[c][tap * 3 + co]; bias [groups][4].
 * Cin % 32 == 0 and Cin <= 320 (P3D_ERR_UNSUPPORTED above: the shared memory holds fewer than two activation tiles). */
int p3d_head_out_conv_f16(const void *in_h16, int B, int H, int W, int in_C, int Cin, int groups, const void *packed_weight,
                          const float *bias, const int32_t *cin0_dev, const int32_t *plane0_dev, const int32_t *cnt_dev,
                          int planes, float *out_nchw, p3d_stream_t stream);
/* The CenterHead's batched ConvModule conv fused with the GEMM of its output convs (the path DenseRPNHead.forward takes
 * when every output conv has <= 3 channels): a 3x3, pad 1 conv of Cout / 64 heads of 64 channels (packed_weight with
 * n_tile 128, scale / shift, ReLU) whose fp16-pair outputs stay in shared memory, where each head's tap-as-N GEMM
 * P[pixel][tap * 3 + co] = sum_c mid[pixel][c] W2[c][tap * 3 + co] runs on them.  packed_w2: per head
 * p3d_dense_conv2d_f16_pack_weights(taps 1, Cin 64, n_tile 32) of W2 (8 KB, heads in Cout order).  Writes p_out
 * [B][Cout / 64][H][W][28] fp32 (columns 0..26 used, 27 zero); status bit 0 as p3d_dense_conv2d_f16.  P is
 * bit-identical to what p3d_head_out_conv_f16 computes from the heads' pixel H16 image.  Cin % 32 == 0 and
 * Cout % 128 == 0 (P3D_ERR_UNSUPPORTED otherwise). */
int p3d_head_conv_p_f16(const void *in_h16, int B, int H, int W, int Cin, const void *packed_weight, int Cout,
                        const float *scale, const float *shift, const void *packed_w2, float *p_out, int32_t *status_dev,
                        p3d_stream_t stream);
/* The output convs from P of p3d_head_conv_p_f16 (groups = Cout / 64): out_nchw[b][plane0[g] + co] = bias[g][co] + the
 * sum of P over the 9 taps, for co < cnt[g] <= 3 (device int32 arrays); bias [groups][4].  Bit-identical to
 * p3d_head_out_conv_f16 on the same heads. */
int p3d_head_tap_sum(const float *p_in, int B, int H, int W, int groups, const float *bias, const int32_t *plane0_dev,
                     const int32_t *cnt_dev, int planes, float *out_nchw, p3d_stream_t stream);
int p3d_dense_conv2d_f16(const void *in_h16, int B, int H, int W, int Cin, const void *packed_weight, int Cout, int n_tile,
                         int kh, int kw, int stride, int pad, int up, const float *scale, const float *shift, int relu,
                         void *out_h16, int out_C, int out_c0, float *out_nchw, int mode, int m_tiles,
                         int32_t *status_dev, p3d_stream_t stream);
/* p3d_dense_conv2d_f16 with a residual (ResNet BasicBlock's conv2 + identity): channels [0, Cout) of the pixel H16 image
 * res_h16 [B, oH, oW, res_C] are added after scale / shift and before ReLU, v = fma(acc, scale, shift) + (hi + lo' 2^-11).
 * res_h16 16-byte aligned and res_C >= Cout (P3D_ERR_INVALID_ARG otherwise); up == 1, H16 output only (out_nchw null),
 * out_c0 % 32 == 0 and res_C % 32 == 0 (P3D_ERR_UNSUPPORTED otherwise). */
int p3d_dense_conv2d_f16_residual(const void *in_h16, int B, int H, int W, int Cin, const void *packed_weight, int Cout,
                                  int n_tile, int kh, int kw, int stride, int pad, int up, const float *scale,
                                  const float *shift, int relu, void *out_h16, int out_C, int out_c0, float *out_nchw,
                                  const void *res_h16, int res_C, int mode, int m_tiles, int32_t *status_dev,
                                  p3d_stream_t stream);
/* Bilinear upsampling (align_corners=True, integer scale s >= 1) of pixel H16 rows in_h16 [B, h, w, C] into channels
 * [out_c0, out_c0 + C) of out_h16 [B, s h, s w, out_C]: Paddle's bilinear_interp_v2 on the merged pair values in fp32
 * (ratio = (in - 1) / (out - 1), h2l (w2l a + w1l b) + h1l (w2l c + w1l d), no contraction), split again; s == 1 copies
 * the pairs.  Status bit 0: an output left fp16's range.  C % 32 == 0 (whole input rows of 32-channel groups),
 * out_c0 % 16 == 0, out_C % 32 == 0,
 * out_c0 + C <= out_C, 16-byte aligned images (P3D_ERR_INVALID_ARG otherwise). */
int p3d_upsample_bilinear_h16(const void *in_h16, int B, int h, int w, int C, int scale, void *out_h16, int out_C, int out_c0,
                              int32_t *status_dev, p3d_stream_t stream);
/* Nearest upsampling (F.interpolate(mode='nearest') to scale x the size, source pixel = output pixel / scale) of pixel
 * H16 rows in_h16 [B, h, w, C] into channels [out_c0, out_c0 + C) of out_h16 [B, scale h, scale w, out_C]: the pairs are
 * copied (exact, no status).  CustomFPN's top-down step writes it as the residual rows of the lateral conv.  Argument
 * contract of p3d_upsample_bilinear_h16 (P3D_ERR_INVALID_ARG otherwise). */
int p3d_upsample_nearest_h16(const void *in_h16, int B, int h, int w, int C, int scale, void *out_h16, int out_C, int out_c0,
                             p3d_stream_t stream);
/* ResNet stem (mmdet ResNet, style 'pytorch'): MaxPool2d(3, 2, 1)(ReLU(conv7x7(in, stride 2, pad 3) * scale[c] +
 * shift[c])) of fp32 NCHW images in [B, 3, H, W], 3 -> 64 channels, into pixel H16 rows out_h16 [B, pH, pW, 64] with
 * cH = (H - 1) / 2 + 1, pH = (cH - 1) / 2 + 1 (the same for W).  Conv on warp MMA with both operands as fp16 pairs
 * (hi.hi + hi.lo' + lo'.hi, fp32 accumulation), BatchNorm (eval) folded into scale / shift [64] by the caller; the pool
 * takes the max in fp32 and the result is split once.  Status bit 0: an input, weight or output left fp16's range.
 * packed_weight: p3d_resnet_stem_packed_weight_bytes() bytes written by p3d_resnet_stem_pack_weights from W [64][3][7][7]
 * fp32 (paddle.nn.Conv2D layout).  Null pointers, B, H, W < 1, packed_weight / out_h16 not 16-byte aligned:
 * P3D_ERR_INVALID_ARG; B > 65535 or B * 3 * H * W >= 2^31: P3D_ERR_UNSUPPORTED. */
size_t p3d_resnet_stem_packed_weight_bytes(void);
int p3d_resnet_stem_pack_weights(const float *weight, void *packed, int32_t *status_dev, p3d_stream_t stream);
int p3d_resnet_stem_h16(const float *in, int B, int H, int W, const void *packed_weight, const float *scale, const float *shift,
                        void *out_h16, int32_t *status_dev, p3d_stream_t stream);
/* BEVDet's test-time image pipeline (PrepareImageInputs.img_transform + mmlabNormalize) of decoded uint8 RGB frames,
 * bit-identical to the host's PIL.Image.resize((rW, rH)) (BICUBIC, 8 bits per channel: fixed-point coefficients with 22
 * fraction bits, horizontal pass rounded and clamped to uint8, then the vertical pass), PIL crop (crop_x, crop_y,
 * crop_x + fW, crop_y + fH) of the resized image (0 outside it) and mmcv.imnormalize: out[n][c][y][x] =
 * fp32(fp64(fp32(v - mean_host[c])) * std_inv_host[c]) with v = the cropped pixel's channel (swap_rb ? 2 - c : c).
 *   frames [N][band_rows][W0][3] uint8: rows [y0, y0 + band_rows) of each H0 x W0 source frame.
 *   kh [rW][kh_size], xbounds [rW][2] = (xmin, n): resized column x = sum over t < n of kh[x][t] * source column xmin + t;
 *   kv [rH][kv_size], ybounds [rH][2] the same for the rows, ymin relative to y0 (ops/image_prep.resize_coeffs; device
 *   int32).  Taps outside the band read 0.  mean_host [3] fp32, std_inv_host [3] fp64: host arrays, copied at the call.
 *   out [N][3][fH][fW] fp32, 16-byte aligned, written in full and nothing else.  No allocation, no host synchronisation.
 * Null pointers, a size < 1, band_rows > H0, |crop| > 2^28, out not 16-byte aligned, or kh_size / kv_size other than
 * Pillow's 2 * ceil(2 * max(in / out, 1)) + 1 for W0 -> rW / H0 -> rH: P3D_ERR_INVALID_ARG.  A reduction by more than 8
 * on either axis (more than 33 taps), N > 65535 or N * 3 * fH * fW >= 2^31: P3D_ERR_UNSUPPORTED. */
int p3d_image_prep_u8(const uint8_t *frames, int N, int band_rows, int H0, int W0, const int32_t *kh, const int32_t *xbounds,
                      int kh_size, int rW, const int32_t *kv, const int32_t *ybounds, int kv_size, int rH, int crop_x,
                      int crop_y, int fH, int fW, const float *mean_host, const double *std_inv_host, int swap_rb,
                      float *out, p3d_stream_t stream);
/* p3d_bev_pool_v2_dev into pixel H16 rows: out_h16 [B, Y, X, out_C] with channel z * c + ch of cell (y, x) (the layout of
 * the planar output, one pixel per row), same accumulation, then split into (hi, lo'); status bit 0 on fp16 overflow.
 * out_h16 is zero-filled here (empty cells and channels >= Z * c).  out_C % 32 == 0 and out_C >= Z * c
 * (P3D_ERR_INVALID_ARG otherwise); c % 4 == 0, c <= 256, feat / out_h16 16-byte aligned, B * Z * Y * X <= 2^31 (the int32
 * ranks' range) (P3D_ERR_UNSUPPORTED). */
int p3d_bev_pool_v2_dev_h16(const float *depth, const float *feat, const int32_t *ranks_depth, const int32_t *ranks_feat,
                            const int32_t *ranks_bev, const int32_t *interval_lengths, const int32_t *interval_starts,
                            const int32_t *counts_dev, int64_t capacity, int c, int B, int Z, int Y, int X, void *out_h16,
                            int out_C, int32_t *status_dev, p3d_stream_t stream);
/* BEVDet4D's shift_feature on pixel H16 rows: channels [0, C) of in_h16 [B, h, w, in_C] resampled at the grid of the
 * affine tf_dev [B, 6] (device fp32, row-major rows 0 and 1 of the 3x3 BEV-pixel transform: g = tf (x, y, 1)),
 * normalised by / (w - 1) * 2 - 1 and sampled as grid_sample(bilinear, padding_mode='zeros', align_corners=True), in fp32
 * without contraction; written to channels [out_c0, out_c0 + C) of out_h16 [B, h, w, out_C].  Taps outside the image
 * (non-finite coordinates included) contribute 0 and are not read.  in_h16 may be out_h16 when the channel ranges are
 * disjoint.  Status bit 0: an output left fp16's range.  C % 16 == 0, C <= in_C, in_C % 32 == 0, out_C % 32 == 0,
 * out_c0 % 16 == 0, out_c0 + C <= out_C, h, w >= 2, 16-byte aligned images (P3D_ERR_INVALID_ARG otherwise). */
int p3d_bev_shift_h16(const void *in_h16, int B, int h, int w, int in_C, int C, const float *tf_dev, void *out_h16, int out_C,
                      int out_c0, int32_t *status_dev, p3d_stream_t stream);

/* SURVEY.md 8f-2: PillarFeatureNet with one PFNLayer
 * (models/voxel_encoders/pillar_encoder.py:156-210, :81-106) fused into one launch: voxels [n, M, F] + counts + coors
 * [n, 4] (b, z, y, x) -> pillar features [n, C].  weight [F + 5, C] (paddle.nn.Linear layout, no bias); BatchNorm1D
 * folded by the caller: y = x * bn_scale[c] + bn_shift[c].  Rows >= *num_voxels_dev (if given) are left untouched. */
int p3d_pillar_feature_net(const float *voxels, const int32_t *num_points_per_voxel, const int32_t *coors,
                           const int32_t *num_voxels_dev, int64_t n_cap, int max_points, int num_point_dim,
                           int out_channels, const float *weight, const float *bn_scale, const float *bn_shift,
                           const float *voxel_size_host, const float *point_cloud_range_host, float *out,
                           p3d_stream_t stream);
/* PillarFeatureNet with two PFNLayers (feat_channels [2 mid, out], as CenterPoint-pillars uses it), fused into one launch:
 * the decoration and padding of p3d_pillar_feature_net, then Linear(F + 5 -> mid) + BN + ReLU per row (weight1
 * [F + 5, mid]), x_max = max over the M rows, Linear over concat([x, x_max]) (weight2 [2 mid, out]: rows 0..mid-1 multiply
 * x, rows mid..2 mid-1 x_max) + BN + ReLU, max over the rows -> [n, out].  Padding rows take part in both maxima.  Both
 * BatchNorm1D folded by the caller.  fp32 FMAs throughout.  mid <= 64 and M <= 64, F <= 8 (P3D_ERR_UNSUPPORTED above). */
int p3d_pillar_feature_net2(const float *voxels, const int32_t *num_points_per_voxel, const int32_t *coors,
                            const int32_t *num_voxels_dev, int64_t n_cap, int max_points, int num_point_dim,
                            int mid_channels, const float *weight1, const float *bn_scale1, const float *bn_shift1,
                            int out_channels, const float *weight2, const float *bn_scale2, const float *bn_shift2,
                            const float *voxel_size_host, const float *point_cloud_range_host, float *out,
                            p3d_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * anchor_head_postprocess      SECOND v1.5 VoxelNet.predict (the path SSDHead.post_process -> rotate_nms_pcdet ports)
 *                              at batch 1 with sigmoid scores and class-agnostic NMS, with no host synchronisation.
 *   head [1, R (C + 9), H, W] fp32 planes, C = num_classes: cls [R x C] | box [R x 7] | dir [R x 2]; channel a * K + k of
 *   each group belongs to anchor (y * W + x) * R + a (K = C, 7, 2).  anchors [A, 7] (x, y, z, w, l, h, theta),
 *   A = H * W * R;  anchor_corners [A, 4] int32 (x_min, y_min, x_max, y_max) clamped voxel indices of each anchor's
 *   near box (16-byte aligned).
 *   coords [coords_cap, 4] (b, z, y, x) of the pillars, *num_coords_dev of them valid (null: all).
 *   Anchors whose occupied-pillar count over the near box is <= anchor_area_threshold are dropped; then
 *   score = max over the classes of sigmoid(cls), label = the first class reaching it; score >= score_threshold,
 *   descending-score order with ties by ascending anchor index, the first nms_pre_max_size, rotated NMS over all
 *   classes together, the first nms_post_max_size kept, direction fix, centre range filter.  num_classes < 1: invalid.
 *   Outputs (device): boxes [nms_post_max_size, 7], scores, labels int64, counts [2] int32 = (score-threshold
 *   candidates, rows written).  Optional (null to skip): anchor_mask [A] uint8, and the decoded candidates in
 *   score order before NMS: sorted_boxes [nms_pre_max_size, 7], sorted_scores [nms_pre_max_size].
 * ------------------------------------------------------------------------------------------- */
size_t p3d_anchor_head_postprocess_workspace_bytes(int num_anchors, int grid_nx, int grid_ny, int nms_pre_max_size);
int p3d_anchor_head_postprocess(const float *head, int feat_h, int feat_w, int anchors_per_loc, int num_classes,
                                const float *anchors, const int32_t *anchor_corners, const int32_t *coords,
                                const int32_t *num_coords_dev, int coords_cap, int grid_nx, int grid_ny,
                                int anchor_area_threshold, float score_threshold,
                                float nms_iou_threshold, int nms_pre_max_size, int nms_post_max_size,
                                const float *post_center_range_host, float *boxes, float *scores, int64_t *labels,
                                int32_t *counts, uint8_t *anchor_mask, float *sorted_boxes, float *sorted_scores,
                                void *workspace, size_t workspace_bytes, p3d_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * merge_sweeps      the multi-sweep input of the nuScenes 10-sweep CenterPoint model on the device: what
 *                   LoadPointCloud.__call__ (paddle3d/transforms/reader.py:116-167) does on the host.
 *   raw       [num_slots, slot_cap, raw_dim] fp32 raw file rows (16-byte aligned, slot_cap % 4 == 0)
 *   desc      [num_entries] device frame descriptor, read by the kernel (one captured graph serves every frame):
 *             entry 0 is the key sweep, then the earlier sweeps in merge order; an entry of 0 rows is empty.
 *   use_dim_host[n_use_dim]  columns kept (n_use_dim == 0: all raw_dim columns); use_time_lag appends fp32(time_lag).
 *   out       [cap, F] fp32, F = (n_use_dim ? n_use_dim : raw_dim) + use_time_lag, fully written: key rows, then the kept
 *             rows of every sweep in input order (the reference's concatenation order), NaN rows from *n_out_dev on.
 *   The key sweep keeps every row, lag 0, no transform.  A sweep drops a row when |c0| < r and |c1| < r (fp32, on the
 *   selected columns 0 and 1); with has_transform its columns 0..2 become fp32(M[0..2] . (c0, c1, c2, 1)) computed in
 *   fp64.  *n_out_dev = min(rows, cap); *status_dev: bit 0 = rows beyond cap were dropped, bit 1 = an entry with a slot
 *   outside [0, num_slots) or rows outside [0, slot_cap] (read as empty).  (raw_dim + F) <= 12.
 * ------------------------------------------------------------------------------------------- */
typedef struct p3d_sweep_desc {
  int32_t slot;             /* slot of `raw` holding this sweep */
  int32_t rows;             /* raw rows in that slot */
  int32_t has_transform;    /* 0: the rows are already in the key frame */
  float time_lag;           /* seconds, the lag column's value */
  double ref_from_curr[12]; /* top three rows of the 4x4 transform into the key frame, row-major */
} p3d_sweep_desc;

size_t p3d_merge_sweeps_workspace_bytes(int num_entries, int64_t slot_cap);
int p3d_merge_sweeps(const float *raw, int num_slots, int64_t slot_cap, int raw_dim, const p3d_sweep_desc *desc,
                     int num_entries, const int32_t *use_dim_host, int n_use_dim, int use_time_lag,
                     float sweep_remove_radius, float *out, int64_t cap, int32_t *n_out_dev, int32_t *status_dev,
                     void *workspace, size_t workspace_bytes, p3d_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Baseline JPEG decode to uint8 RGB rows, bit-identical to libjpeg-turbo's C paths (jpeg_idct_islow, fancy upsampling,
 * ycc_rgb_convert) that PIL.Image.open runs.  Supported: SOF0 / SOF1 Huffman DCT, 8-bit, three components Y Cb Cr in
 * one interleaved scan, chroma 1x1 and luma 1x1, 2x1 or 2x2, any restart interval and tables.  The host reads the
 * markers (paddle3d_b200/ops/jpeg.parse) and fills one p3d_jpeg_desc per image; every size, offset and table is read on
 * the device, so a captured graph serves any compressed lengths and tables.
 *   data [data_bytes] uint8: the concatenated files; desc [N] (device).  Every image is H x W (desc->height / width).
 *   out [N][y1 - y0][W][3] uint8: rows [y0, y1) of every image.  status_dev [N] int32 (device), one word per image:
 *   bits are OR-ed in and never cleared here: 1 = an undefined Huffman code or a run past coefficient 63, 2 = a restart marker out of
 *   sequence, missing or misplaced, 4 = the data ends before the last MCU, 8 = a marker other than RSTn (or a fill byte)
 *   in the entropy-coded segment, 16 = a descriptor disagrees with the call (size, sampling, a segment outside data or
 *   longer than max_bytes; that image is not decoded).  Corrupt data never reads outside its segment.
 *   workspace: p3d_jpeg_decode_workspace_bytes(N, H, W, max_bytes) bytes, max_bytes = the largest entropy-coded
 *   segment.  No allocation, no host synchronisation.
 * Null pointers, a size < 1 or rows outside [0, H): P3D_ERR_INVALID_ARG.  N > 64, H or W > 8192 or max_bytes > 2^28:
 * P3D_ERR_UNSUPPORTED.
 * ------------------------------------------------------------------------------------------- */
#define P3D_JPEG_MAX_IMAGES 64
#define P3D_JPEG_MAX_SIDE 8192
typedef struct p3d_jpeg_desc {
  int64_t offset;            /* first byte of the entropy-coded segment in data */
  int32_t length;            /* its bytes, up to the EOI marker */
  int32_t height, width;
  int32_t hs, vs;            /* luma sampling factors (chroma 1 x 1) */
  int32_t restart_interval;  /* MCUs per restart interval, 0 = none */
  uint16_t quant[3][64];     /* per component, natural order */
  uint8_t dc_bits[3][16], dc_vals[3][16], ac_bits[3][16], ac_vals[3][256]; /* per component: BITS / HUFFVAL */
} p3d_jpeg_desc;

size_t p3d_jpeg_decode_workspace_bytes(int N, int H, int W, int64_t max_bytes);
int p3d_jpeg_decode_u8(const uint8_t *data, int64_t data_bytes, const p3d_jpeg_desc *desc, int N, int H, int W, int y0,
                       int y1, int64_t max_bytes, uint8_t *out, int32_t *status_dev, void *workspace,
                       size_t workspace_bytes, p3d_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * BEVFusion (bevf_pp) entry points.  PARITY UNPINNED: recalled from mmdet3d v0.17 (HardVFE, Anchor3DHead,
 * box3d_multiclass_nms) and ADLab's BEVFusion (SE_Block), not checked against either.
 *
 * p3d_hard_vfe: mmdet3d HardVFE(feat_channels [mid, out], with_cluster_center, with_voxel_center, no distance) as one
 * launch, the two-layer kernel of p3d_pillar_feature_net2 with a wider decoration: per point the F raw values, xyz minus
 * the pillar mean, xyz minus the voxel centre (coors * voxel_size + voxel_size / 2 + range_min, z included), F + 6
 * features; padding rows zeroed; VFELayer 0 = Linear(F + 6 -> mid) + BN + ReLU concatenated with its max over the M rows
 * (weight1 [F + 6, mid]; mid is not halved), VFELayer 1 = Linear(2 mid -> out) + BN + ReLU, max over the rows -> [n, out].
 * voxel_size_host / point_cloud_range_host: 3 / 6 values.  Limits of p3d_pillar_feature_net2.
 *
 * p3d_se_gate_h16: BEVFusion's SE_Block on a pixel H16 image img_h16 [B, H, W, C] in place:
 *   gate[b, o] = sigmoid(bias[o] + sum_c weight[o, c] * mean_hw(img[b, :, :, c])), x *= gate[b, c].
 *   The mean: per-CTA partial sums in fp64, then summed in index order (no atomics: bit-reproducible).  The gate is
 *   computed in fp64 and rounded to fp32 into gate_dev [B, C] (device).  The scale rebuilds each value from its pair in
 *   fp32, multiplies by the fp32 gate and splits again; status bit 0 as p3d_dense_conv2d_f16.  weight [C, C] (the 1x1
 *   conv's [out, in]), bias [C], device fp32.  C % 32 == 0, 16-byte aligned image (P3D_ERR_INVALID_ARG otherwise);
 *   C <= 1024, B <= 65535 (P3D_ERR_UNSUPPORTED above).  workspace: p3d_se_gate_workspace_bytes(B, H, W, C).
 *
 * p3d_anchor3d_postprocess: Anchor3DHead.get_bboxes_single + box3d_multiclass_nms at batch 1, sigmoid scores, every
 * class in the same launches, no host synchronisation.
 *   head [R (C + 9 + 2), H, W] fp32 planes: cls [R x C] | reg [R x 9] | dir [R x 2]; channel a * K + k of a group belongs
 *   to anchor (y * W + x) * R + a.  anchors [A, 9] (x, y, z, w, l, h, r, vx, vy), A = H * W * R.
 *   1. score = max over the classes of sigmoid(cls) (NaN when a class is NaN); dir = argmax of the two dir logits, a tie
 *      to bin 0.
 *   2. A > nms_pre: the nms_pre anchors of highest score, in descending score order, ties by the lower anchor index, a
 *      NaN score above every number (torch.topk's order).  A <= nms_pre: every anchor, in anchor order.  Only anchors
 *      that can reach the output (a class score > score_thr, or a NaN score) are ranked: the others cannot enter the
 *      output and rank below every one that can.
 *   3. DeltaXYZWLHRBBoxCoder.decode: za += ha / 2, diag = sqrt(la^2 + wa^2), x = xt diag + xa, y = yt diag + ya,
 *      z = zt ha + za, (w, l, h) = exp(t) * anchor, r = rt + ra, z -= h / 2, (vx, vy) = t + anchor; fp32, every
 *      operation rounded on its own.
 *   4. per class c in order: the kept anchors with sigmoid(cls_c) > score_thr, greedy NMS in descending class score
 *      (ties by kept order) with suppression at BEV IoU > nms_thr, the IoU of box_geom.cuh on (x, y, w, l, r) taken
 *      as (x, y, dx, dy, heading).  Which rotation convention the reference's NMS applies is unpinned.
 *   5. more than max_num survivors over all classes: sorted by score, descending, ties in class-major order, the first
 *      max_num kept; otherwise class-major order.
 *   6. r = limit_period(r - dir_offset, dir_limit_offset, pi) + dir_offset + pi * dir, limit_period(v, o, p) =
 *      v - floor(v / p + o) * p in fp32.
 *   Outputs (device): boxes [max_num, 9], scores [max_num], labels int64 [max_num], count [1] int32 (rows written).
 *   Limits (P3D_ERR_UNSUPPORTED): C <= 64, A < 2^31, nms_pre <= 4096.  workspace: p3d_anchor3d_postprocess_workspace_bytes.
 * ------------------------------------------------------------------------------------------- */
int p3d_hard_vfe(const float *voxels, const int32_t *num_points_per_voxel, const int32_t *coors,
                 const int32_t *num_voxels_dev, int64_t n_cap, int max_points, int num_point_dim, int mid_channels,
                 const float *weight1, const float *bn_scale1, const float *bn_shift1, int out_channels,
                 const float *weight2, const float *bn_scale2, const float *bn_shift2, const float *voxel_size_host,
                 const float *point_cloud_range_host, float *out, p3d_stream_t stream);
size_t p3d_se_gate_workspace_bytes(int B, int H, int W, int C);
int p3d_se_gate_h16(void *img_h16, int B, int H, int W, int C, const float *weight, const float *bias, float *gate_dev,
                    int32_t *status_dev, void *workspace, size_t workspace_bytes, p3d_stream_t stream);
size_t p3d_anchor3d_postprocess_workspace_bytes(int feat_h, int feat_w, int anchors_per_loc, int num_classes,
                                                int nms_pre, int max_num);
int p3d_anchor3d_postprocess(const float *head, int feat_h, int feat_w, int anchors_per_loc, int num_classes,
                             const float *anchors, int nms_pre, float score_thr, float nms_thr, int max_num,
                             float dir_offset, float dir_limit_offset, float *boxes, float *scores, int64_t *labels,
                             int32_t *count, void *workspace, size_t workspace_bytes, p3d_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* P3D_B200_H_ */
