// iou3d_nms ops for sm_90a: pairwise BEV overlap / IoU and sync-free rotated / axis-aligned NMS.
// Replaces paddle3d/ops/iou3d_nms/iou3d_nms.cpp:44-204 + iou3d_nms_kernel.cu:275-482.
#include "box_geom.cuh"
#include "common.cuh"
#include "nms_reduce.cuh"

namespace p3d {
namespace {

constexpr int kPairTile = 16;

// One thread per (a, b) pair; the 16 b-boxes of a tile are staged in shared memory once.
template <bool kIou>
__global__ void __launch_bounds__(kPairTile *kPairTile) pairwise_kernel(int na, const float *__restrict__ A, int nb,
                                                                        const float *__restrict__ B,
                                                                        float *__restrict__ out) {
  __shared__ float sa[kPairTile * 7], sb[kPairTile * 7];
  const int tid = threadIdx.y * kPairTile + threadIdx.x;
  const int a0 = blockIdx.y * kPairTile, b0 = blockIdx.x * kPairTile;
  if (tid < kPairTile * 7) {
    const int r = tid / 7;
    sa[tid] = (a0 + r < na) ? A[static_cast<size_t>(a0) * 7 + tid] : 0.f;
    sb[tid] = (b0 + r < nb) ? B[static_cast<size_t>(b0) * 7 + tid] : 0.f;
  }
  __syncthreads();
  const int ai = a0 + threadIdx.y, bi = b0 + threadIdx.x;
  if (ai >= na || bi >= nb) return;
  const float *pa = sa + threadIdx.y * 7, *pb = sb + threadIdx.x * 7;
  out[static_cast<size_t>(ai) * nb + bi] = kIou ? geom::iou_rotated(pa, pb) : geom::overlap_area(pa, pb);
}

// Suppression bit-matrix, upper triangle only: block (cb, rb) with cb >= rb, 64 threads = 64 rows.
template <bool kNormal>
__global__ void __launch_bounds__(64) nms_mask_kernel(int n, float thr, const float *__restrict__ boxes,
                                                      unsigned long long *__restrict__ mask) {
  const int rb = blockIdx.y, cb = blockIdx.x;
  if (cb < rb) return;
  const int rows = min(n - rb * 64, 64), cols = min(n - cb * 64, 64);
  __shared__ float s_col[64 * 7], s_row[64 * 7];
  __shared__ unsigned short s_pairs[64 * 64];
  __shared__ unsigned long long s_bits[64];
  __shared__ int s_cnt[3];
  for (int k = threadIdx.x; k < cols * 7; k += 64) s_col[k] = boxes[static_cast<size_t>(cb) * 64 * 7 + k];
  for (int k = threadIdx.x; k < rows * 7; k += 64) s_row[k] = boxes[static_cast<size_t>(rb) * 64 * 7 + k];
  __syncthreads();
  unsigned long long t = 0ull;
  if (kNormal) {
    if (threadIdx.x < rows) {
      const int start = (rb == cb) ? threadIdx.x + 1 : 0;
      for (int j = start; j < cols; ++j)
        if (geom::iou_axis_aligned(s_row + threadIdx.x * 7, s_col + j * 7) > thr) t |= 1ull << j;
    }
  } else {
    t = nms_rotated_tile(s_row, s_col, rows, cols, rb == cb, thr, s_pairs, s_bits, s_cnt);
  }
  if (threadIdx.x < rows) mask[static_cast<size_t>(rb * 64 + threadIdx.x) * ((n + 63) / 64) + cb] = t;
}

__global__ void __launch_bounds__(256) nms_reduce_kernel(const unsigned long long *__restrict__ mask, int n,
                                                         int32_t *__restrict__ keep, int32_t *__restrict__ num_keep) {
  extern __shared__ unsigned long long s_dyn[];
  __shared__ unsigned long long s_misc[2];
  const int k = nms_greedy_cta(mask, n, (n + 63) / 64, keep, s_dyn, s_misc);
  if (threadIdx.x == 0) num_keep[0] = k;
}

}  // namespace
}  // namespace p3d

using namespace p3d;

static int pairwise(const float *a, int na, const float *b, int nb, float *out, bool iou, p3d_stream_t stream) {
  if (na < 0 || nb < 0 || ((na && nb) && (!a || !b || !out))) return P3D_ERR_INVALID_ARG;
  if (na == 0 || nb == 0) return P3D_OK;
  dim3 grid(div_up(nb, kPairTile), div_up(na, kPairTile)), block(kPairTile, kPairTile);
  if (grid.y > 65535) return P3D_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (iou)
    pairwise_kernel<true><<<grid, block, 0, st>>>(na, a, nb, b, out);
  else
    pairwise_kernel<false><<<grid, block, 0, st>>>(na, a, nb, b, out);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" int p3d_boxes_overlap_bev(const float *boxes_a, int num_a, const float *boxes_b, int num_b,
                                     float *overlap, p3d_stream_t stream) {
  return pairwise(boxes_a, num_a, boxes_b, num_b, overlap, false, stream);
}

extern "C" int p3d_boxes_iou_bev(const float *boxes_a, int num_a, const float *boxes_b, int num_b, float *iou,
                                 p3d_stream_t stream) {
  return pairwise(boxes_a, num_a, boxes_b, num_b, iou, true, stream);
}

extern "C" size_t p3d_nms_workspace_bytes(int n) {
  if (n < 0) return 0;
  const size_t cb = (static_cast<size_t>(n) + 63) / 64;
  return align_up(static_cast<size_t>(n > 0 ? n : 1) * (cb ? cb : 1) * sizeof(unsigned long long));
}

extern "C" int p3d_nms(const float *boxes, int n, float nms_overlap_thresh, int normal, int32_t *keep,
                       int32_t *num_keep, void *workspace, size_t workspace_bytes, p3d_stream_t stream) {
  if (n < 0 || !num_keep || (n && (!boxes || !keep || !workspace))) return P3D_ERR_INVALID_ARG;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (n == 0) {
    P3D_CUDA_CHECK(cudaMemsetAsync(num_keep, 0, sizeof(int32_t), st));
    return P3D_OK;
  }
  if (workspace_bytes < p3d_nms_workspace_bytes(n)) return P3D_ERR_WORKSPACE;
  const int cb = (n + 63) / 64;
  if (cb > 65535) return P3D_ERR_UNSUPPORTED;
  if (static_cast<size_t>(cb) * 8 > 200 * 1024) return P3D_ERR_UNSUPPORTED;
  unsigned long long *mask = static_cast<unsigned long long *>(workspace);
  dim3 grid(cb, cb);
  if (normal)
    nms_mask_kernel<true><<<grid, 64, 0, st>>>(n, nms_overlap_thresh, boxes, mask);
  else
    nms_mask_kernel<false><<<grid, 64, 0, st>>>(n, nms_overlap_thresh, boxes, mask);
  P3D_LAUNCH_CHECK();
  const size_t smem = static_cast<size_t>(cb) * sizeof(unsigned long long);
  if (smem > 48 * 1024)
    P3D_CUDA_CHECK(cudaFuncSetAttribute(nms_reduce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(smem)));
  nms_reduce_kernel<<<1, 256, smem, st>>>(mask, n, keep, num_keep);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
