// Anchor (SSD) head postprocess for sm_90a: SECOND v1.5 VoxelNet.predict at batch 1, no host synchronisation
// (every count stays on the device, buffers are sized by capacity), so a frame can be captured in a CUDA graph.
//
// The reference runs this in Python (SSDHead.post_process -> rotate_nms_pcdet): masked_select (D2H sync), argsort, the
// iou3d_nms op with its D2H of the bit-matrix and host greedy loop, gathers.  Here:
//   A1 ahp_occ        occupied-pillar count per BEV cell from the pillar coords (sparse_sum_for_anchors_mask)
//   A2 ahp_col/row    2-D inclusive prefix sum of that map (cumsum(0).cumsum(1)), integers: exact in any order
//   A3 ahp_score      per anchor: area = ID - IB - IC + IA on its four (host-precomputed) clamped voxel corners
//                     (fused_get_anchors_area), keep area > thr; score = max over the C classes of sigmoid(cls_c)
//                     (encode_background_as_zeros, use_multi_class_nms off; NaN if any class is NaN); candidate if
//                     score >= thr;
//                     51-bit sort key (~score_bits << 20 | anchor) - descending score, ties by ascending anchor index
//   A4 cub radix sort of the keys (non-candidates carry the all-ones key and sink to the end)
//   A5 ahp_gather     first min(candidates, pre_max): class label (recomputed, so no per-anchor label array),
//                     second_box_decode, dir argmax, NMS box laid out as rotate_nms_pcdet does:
//                     (x, y, z, l, w, h, -theta - pi/2) in fp32.  NMS is class-agnostic, as in the reference
//   A6 rotated-IoU bit-matrix, one thread per pair (box_geom.cuh) + A7 on-device greedy pass (nms_reduce.cuh), stopping
//                     at post_max kept boxes
//   A8 ahp_emit       direction fix ((theta > 0) xor dir -> theta + pi), centre range filter, order-preserving compaction
// The fp32 expressions of A3 / A5 / A8 are written with explicit roundings (no FMA contraction) so that the numpy
// restatement in oracle/pointpillars.py computes the same values.
#include <cub/cub.cuh>

#include "box_geom.cuh"
#include "common.cuh"
#include "nms_reduce.cuh"

namespace p3d {
namespace {

constexpr int kIdxBits = 20;                         // anchor index bits of a sort key: A < 2^20 - 1
constexpr int kKeyBits = 31 + kIdxBits;              // score part: 0x7fffffff - bits(score), score >= 0
constexpr unsigned long long kNoKey = (1ull << kKeyBits) - 1;
constexpr float kHalfPi = 1.57079637f;               // fp32(pi / 2), as paddle rounds the python scalar
constexpr float kPi = 3.14159274f;                   // fp32(pi)

struct AhpAttrs {
  int A, HW, R, C, nx, ny, area_thr, pre_max, post_max, cbmax, coords_cap;
  float score_thr, iou_thr;
  float lo[3], hi[3];  // post_center_limit_range
};

struct AhpWs {
  int32_t *occ;               // [ny * nx] occupancy
  int32_t *sum;               // [ny * nx] its 2-D inclusive prefix sum
  int32_t *cnt;               // [0] candidates, [1] boxes kept by the greedy pass
  unsigned long long *keys;   // [A]
  unsigned long long *sorted; // [A]
  void *cub_tmp;
  size_t cub_bytes;
  float *top_box;             // [pre_max, 7] decoded boxes in score order
  float *top_score;           // [pre_max]
  int32_t *top_dir;           // [pre_max]
  int32_t *top_label;         // [pre_max]
  float *nms_box;             // [pre_max, 7]
  unsigned long long *mask;   // [pre_max, cbmax]
  int32_t *keep;              // [pre_max]
  size_t bytes;
};

AhpWs carve(void *p, int A, int cells, int pre_max) {
  AhpWs w;
  Carver c(p);
  const int cbmax = (pre_max + 63) / 64;
  w.occ = c.take<int32_t>(static_cast<size_t>(cells));
  w.sum = c.take<int32_t>(static_cast<size_t>(cells));
  w.cnt = c.take<int32_t>(2);
  w.keys = c.take<unsigned long long>(A);
  w.sorted = c.take<unsigned long long>(A);
  w.cub_bytes = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, w.cub_bytes, static_cast<const unsigned long long *>(nullptr),
                                 static_cast<unsigned long long *>(nullptr), A, 0, kKeyBits);
  w.cub_tmp = c.take<char>(w.cub_bytes);
  w.top_box = c.take<float>(static_cast<size_t>(pre_max) * 7);
  w.top_score = c.take<float>(pre_max);
  w.top_dir = c.take<int32_t>(pre_max);
  w.top_label = c.take<int32_t>(pre_max);
  w.nms_box = c.take<float>(static_cast<size_t>(pre_max) * 7);
  w.mask = c.take<unsigned long long>(static_cast<size_t>(pre_max) * cbmax);
  w.keep = c.take<int32_t>(pre_max);
  w.bytes = c.off;
  return w;
}

__device__ __forceinline__ float sigmoid_f32(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }

// Score and label of one anchor: max over the C class planes of sigmoid(cls_c), label = the first class reaching it.
// The comparison is on the fp32 sigmoid values (as the reference's max / argmax over sigmoid(cls)), not on the logits:
// two logits may round to the same score, and then the lower class wins.  A NaN logit in any class makes the score NaN
// (labelled with the first NaN class), as the reference's max propagates it, so the anchor is never a candidate.
// cls points at class 0 of the anchor's group.
__device__ __forceinline__ float class_max(const float *__restrict__ cls, size_t HW, int C, int &label) {
  float best = sigmoid_f32(cls[0]);
  label = 0;
  for (int c = 1; c < C && best == best; ++c) {
    const float s = sigmoid_f32(cls[static_cast<size_t>(c) * HW]);
    if (s > best || s != s) {
      best = s;
      label = c;
    }
  }
  return best;
}

// coords [cap, 4] (b, z, y, x) of the pillars; one pillar per cell, the count is still a sum as in the reference
__global__ void __launch_bounds__(256) ahp_occ_kernel(const int32_t *__restrict__ coords, const int32_t *__restrict__ n_dev,
                                                      AhpAttrs at, AhpWs w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = n_dev ? min(n_dev[0], at.coords_cap) : at.coords_cap;
  if (i >= n) return;
  const int4 c = *reinterpret_cast<const int4 *>(coords + static_cast<size_t>(i) * 4);
  if (c.z < 0 || c.z >= at.ny || c.w < 0 || c.w >= at.nx) return;
  atomicAdd(&w.occ[c.z * at.nx + c.w], 1);
}

// cumsum over y: one thread per column (coalesced across the warp), occ -> sum.  Separate source and destination let
// the unrolled loads of a column issue together instead of one L2 round trip per row.
__global__ void __launch_bounds__(256) ahp_col_scan_kernel(AhpAttrs at, const int32_t *__restrict__ occ,
                                                           int32_t *__restrict__ sum) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= at.nx) return;
  int acc = 0;
#pragma unroll 16
  for (int y = 0; y < at.ny; ++y) {
    acc += __ldg(occ + y * at.nx + x);
    sum[y * at.nx + x] = acc;
  }
}

// cumsum over x: one warp per row, 32 cells per step
__global__ void __launch_bounds__(256) ahp_row_scan_kernel(AhpAttrs at, AhpWs w) {
  const int y = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (y >= at.ny) return;
  int32_t *row = w.sum + static_cast<size_t>(y) * at.nx;
  int carry = 0;
  for (int x0 = 0; x0 < at.nx; x0 += 32) {
    const int x = x0 + lane;
    int v = x < at.nx ? row[x] : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, v, d);
      if (lane >= d) v += t;
    }
    if (x < at.nx) row[x] = v + carry;
    carry += __shfl_sync(0xffffffffu, v, 31);
  }
}

// anchor_corners [A, 4] int32: (x_min, y_min, x_max, y_max) voxel indices, clamped to the grid
__global__ void __launch_bounds__(256) ahp_score_kernel(const float *__restrict__ head, const int4 *__restrict__ corners,
                                                        AhpAttrs at, AhpWs w, uint8_t *__restrict__ mask_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool cand = false;
  unsigned long long key = kNoKey;
  if (i < at.A) {
    const int4 c = corners[i];
    const int32_t *S = w.sum;
    const int nx = at.nx;
    const int area = S[c.w * nx + c.z] - S[c.w * nx + c.x] - S[c.y * nx + c.z] + S[c.y * nx + c.x];
    const bool keep = area > at.area_thr;
    if (mask_out) mask_out[i] = keep ? 1 : 0;
    if (keep) {
      const int cell = i / at.R, a = i - cell * at.R;
      int label;
      const float s = class_max(head + static_cast<size_t>(a) * at.C * at.HW + cell, at.HW, at.C, label);
      cand = s >= at.score_thr;
      key = (static_cast<unsigned long long>(0x7fffffffu - __float_as_uint(s)) << kIdxBits) | static_cast<unsigned>(i);
    }
    w.keys[i] = cand ? key : kNoKey;
  }
  const unsigned m = __ballot_sync(0xffffffffu, cand);
  if (m && (threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(&w.cnt[0], __popc(m));
}

__global__ void __launch_bounds__(128) ahp_gather_kernel(const float *__restrict__ head, const float *__restrict__ anchors,
                                                         AhpAttrs at, AhpWs w, float *__restrict__ dbg_boxes,
                                                         float *__restrict__ dbg_scores) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = min(w.cnt[0], at.pre_max);
  if (r >= n) return;
  const int i = static_cast<int>(w.sorted[r] & ((1ull << kIdxBits) - 1));
  const int cell = i / at.R, a = i - cell * at.R;
  const size_t HW = at.HW;
  const float *an = anchors + static_cast<size_t>(i) * 7;
  const float xa = an[0], ya = an[1], wa = an[3], la = an[4], ha = an[5], ra = an[6];
  const float *bt = head + (static_cast<size_t>(at.R) * at.C + a * 7) * HW + cell;
  const float xt = bt[0], yt = bt[HW], zt = bt[2 * HW], wt = bt[3 * HW], lt = bt[4 * HW], ht = bt[5 * HW], rt = bt[6 * HW];
  // second_box_decode (no smooth_dim, no angle vector)
  const float za = __fadd_rn(an[2], __fmul_rn(ha, 0.5f));
  const float diag = __fsqrt_rn(__fadd_rn(__fmul_rn(la, la), __fmul_rn(wa, wa)));
  float b[7];
  b[0] = __fadd_rn(__fmul_rn(xt, diag), xa);
  b[1] = __fadd_rn(__fmul_rn(yt, diag), ya);
  b[3] = __fmul_rn(expf(wt), wa);
  b[4] = __fmul_rn(expf(lt), la);
  b[5] = __fmul_rn(expf(ht), ha);
  b[2] = __fsub_rn(__fadd_rn(__fmul_rn(zt, ha), za), __fmul_rn(b[5], 0.5f));
  b[6] = __fadd_rn(rt, ra);
  const float *dt = head + (static_cast<size_t>(at.C + 7) * at.R + a * 2) * HW + cell;
  const int dir = dt[HW] > dt[0] ? 1 : 0;  // argmax, ties to index 0
  int label;
  const float s = class_max(head + static_cast<size_t>(a) * at.C * HW + cell, HW, at.C, label);
  float *tb = w.top_box + static_cast<size_t>(r) * 7;
#pragma unroll
  for (int k = 0; k < 7; ++k) tb[k] = b[k];
  w.top_score[r] = s;
  w.top_dir[r] = dir;
  w.top_label[r] = label;
  float *nb = w.nms_box + static_cast<size_t>(r) * 7;  // rotate_nms_pcdet: columns (0, 1, 2, 4, 3, 5), -theta - pi/2
  nb[0] = b[0];
  nb[1] = b[1];
  nb[2] = b[2];
  nb[3] = b[4];
  nb[4] = b[3];
  nb[5] = b[5];
  nb[6] = __fsub_rn(-b[6], kHalfPi);
  if (dbg_boxes) {
#pragma unroll
    for (int k = 0; k < 7; ++k) dbg_boxes[static_cast<size_t>(r) * 7 + k] = b[k];
  }
  if (dbg_scores) dbg_scores[r] = s;
}

// Suppression bit-matrix, one thread per box pair: warp (i, h) evaluates row i against columns 32 h .. 32 h + 31 and
// writes that half of mask word [i][h / 2] with one ballot.  The top candidates of an anchor head crowd into a few
// regions, so most pairs survive the cheap reject and a 64 x 64 tile per 64-thread CTA (nms_rotated_tile) would leave the
// GPU nearly idle.  Same bits as the tile: geom::iou_rotated(box i, box j) > thr for j > i, zero elsewhere, after the
// same exact reject (centres farther apart than the half diagonals + slack cannot overlap: IoU 0).
__global__ void __launch_bounds__(256) ahp_nms_mask_kernel(AhpAttrs at, AhpWs w) {
  const int n = min(w.cnt[0], at.pre_max);
  const int halves = 2 * at.cbmax;
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= static_cast<long long>(n) * halves) return;
  const int i = static_cast<int>(warp / halves), h = static_cast<int>(warp - static_cast<long long>(i) * halves);
  const int j = h * 32 + lane;
  bool sup = false;
  if (j > i && j < n) {
    const float *a = w.nms_box + static_cast<size_t>(i) * 7, *b = w.nms_box + static_cast<size_t>(j) * 7;
    const float dx = a[0] - b[0], dy = a[1] - b[1];
    const float R = 0.5f * sqrtf(a[3] * a[3] + a[4] * a[4]) + 0.5f * sqrtf(b[3] * b[3] + b[4] * b[4]) + 0.1f;
    if (at.iou_thr < 0.f || dx * dx + dy * dy <= R * R * 1.001f) sup = geom::iou_rotated(a, b) > at.iou_thr;
  }
  const unsigned bits = __ballot_sync(0xffffffffu, sup);
  if (lane == 0) reinterpret_cast<unsigned *>(w.mask)[static_cast<size_t>(i) * halves + h] = bits;  // little-endian halves
}

__global__ void __launch_bounds__(256) ahp_greedy_kernel(AhpAttrs at, AhpWs w) {
  extern __shared__ unsigned long long s_dyn[];
  __shared__ unsigned long long s_misc[2];
  const int n = min(w.cnt[0], at.pre_max);
  const int k = nms_greedy_cta(w.mask, n, at.cbmax, w.keep, s_dyn, s_misc, at.post_max);
  if (threadIdx.x == 0) w.cnt[1] = k;
}

__global__ void __launch_bounds__(256) ahp_emit_kernel(AhpAttrs at, AhpWs w, float *__restrict__ boxes,
                                                       float *__restrict__ scores, long long *__restrict__ labels,
                                                       int32_t *__restrict__ counts) {
  __shared__ int s_warp[8];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int n = min(w.cnt[1], at.post_max);
  int base = 0;
  for (int r0 = 0; r0 < n; r0 += 256) {
    const int r = r0 + tid;
    bool ok = false;
    float b[7];
    float s = 0.f;
    int label = 0;
    if (r < n) {
      const int j = w.keep[r];
      const float *tb = w.top_box + static_cast<size_t>(j) * 7;
#pragma unroll
      for (int k = 0; k < 7; ++k) b[k] = tb[k];
      if ((b[6] > 0.f) != (w.top_dir[j] != 0)) b[6] = __fadd_rn(b[6], kPi);
      s = w.top_score[j];
      label = w.top_label[j];
      ok = b[0] >= at.lo[0] && b[1] >= at.lo[1] && b[2] >= at.lo[2] && b[0] <= at.hi[0] && b[1] <= at.hi[1] &&
           b[2] <= at.hi[2];
    }
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_warp[wid] = __popc(m);
    __syncthreads();
    int off = base + __popc(m & ((1u << lane) - 1));
    int total = 0;
    for (int k = 0; k < 8; ++k) {
      if (k < wid) off += s_warp[k];
      total += s_warp[k];
    }
    if (ok) {
#pragma unroll
      for (int k = 0; k < 7; ++k) boxes[static_cast<size_t>(off) * 7 + k] = b[k];
      scores[off] = s;
      labels[off] = label;
    }
    base += total;
    __syncthreads();
  }
  if (tid == 0) {
    counts[0] = w.cnt[0];
    counts[1] = base;
  }
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" size_t p3d_anchor_head_postprocess_workspace_bytes(int num_anchors, int grid_nx, int grid_ny, int nms_pre_max_size) {
  if (num_anchors < 1 || num_anchors >= (1 << kIdxBits) - 1 || grid_nx < 1 || grid_ny < 1 || nms_pre_max_size < 1)
    return 0;
  return carve(nullptr, num_anchors, grid_nx * grid_ny, nms_pre_max_size).bytes;
}

extern "C" int p3d_anchor_head_postprocess(const float *head, int feat_h, int feat_w, int anchors_per_loc, int num_classes,
                                           const float *anchors, const int32_t *anchor_corners, const int32_t *coords,
                                           const int32_t *num_coords_dev, int coords_cap, int grid_nx, int grid_ny,
                                           int anchor_area_threshold, float score_threshold, float nms_iou_threshold,
                                           int nms_pre_max_size,
                                           int nms_post_max_size, const float *post_center_range_host, float *boxes,
                                           float *scores, int64_t *labels, int32_t *counts, uint8_t *anchor_mask,
                                           float *sorted_boxes, float *sorted_scores, void *workspace,
                                           size_t workspace_bytes, p3d_stream_t stream) {
  if (!head || !anchors || !anchor_corners || !post_center_range_host || !boxes || !scores || !labels || !counts ||
      !workspace || feat_h < 1 || feat_w < 1 || anchors_per_loc < 1 || num_classes < 1 || coords_cap < 0 ||
      (coords_cap && !coords) || grid_nx < 1 || grid_ny < 1 || nms_pre_max_size < 1 || nms_post_max_size < 1 ||
      score_threshold < 0.f)
    return P3D_ERR_INVALID_ARG;
  if ((reinterpret_cast<uintptr_t>(anchor_corners) & 15) || (reinterpret_cast<uintptr_t>(coords) & 15))
    return P3D_ERR_INVALID_ARG;
  const long long A = static_cast<long long>(feat_h) * feat_w * anchors_per_loc;
  if (A >= (1 << kIdxBits) - 1) return P3D_ERR_UNSUPPORTED;
  const int cbmax = (nms_pre_max_size + 63) / 64;
  if (static_cast<size_t>(cbmax) * 8 > 48 * 1024) return P3D_ERR_UNSUPPORTED;
  AhpWs w = carve(workspace, static_cast<int>(A), grid_nx * grid_ny, nms_pre_max_size);
  if (workspace_bytes < w.bytes) return P3D_ERR_WORKSPACE;
  AhpAttrs at;
  at.A = static_cast<int>(A);
  at.HW = feat_h * feat_w;
  at.R = anchors_per_loc;
  at.C = num_classes;
  at.nx = grid_nx;
  at.ny = grid_ny;
  at.area_thr = anchor_area_threshold;
  at.pre_max = nms_pre_max_size;
  at.post_max = nms_post_max_size;
  at.cbmax = cbmax;
  at.coords_cap = coords_cap;
  at.score_thr = score_threshold;
  at.iou_thr = nms_iou_threshold;
  for (int k = 0; k < 3; ++k) {
    at.lo[k] = post_center_range_host[k];
    at.hi[k] = post_center_range_host[3 + k];
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  P3D_CUDA_CHECK(cudaMemsetAsync(w.occ, 0, sizeof(int32_t) * static_cast<size_t>(grid_nx) * grid_ny, st));
  P3D_CUDA_CHECK(cudaMemsetAsync(w.cnt, 0, sizeof(int32_t) * 2, st));
  if (coords_cap > 0) {
    ahp_occ_kernel<<<div_up(coords_cap, 256), 256, 0, st>>>(coords, num_coords_dev, at, w);
    P3D_LAUNCH_CHECK();
  }
  ahp_col_scan_kernel<<<div_up(grid_nx, 64), 64, 0, st>>>(at, w.occ, w.sum);
  P3D_LAUNCH_CHECK();
  ahp_row_scan_kernel<<<div_up(static_cast<long long>(grid_ny) * 32, 256), 256, 0, st>>>(at, w);
  P3D_LAUNCH_CHECK();
  ahp_score_kernel<<<div_up(A, 256), 256, 0, st>>>(head, reinterpret_cast<const int4 *>(anchor_corners), at, w, anchor_mask);
  P3D_LAUNCH_CHECK();
  size_t tmp = w.cub_bytes;
  P3D_CUDA_CHECK(cub::DeviceRadixSort::SortKeys(w.cub_tmp, tmp, w.keys, w.sorted, static_cast<int>(A), 0, kKeyBits, st));
  ahp_gather_kernel<<<div_up(nms_pre_max_size, 128), 128, 0, st>>>(head, anchors, at, w, sorted_boxes, sorted_scores);
  P3D_LAUNCH_CHECK();
  ahp_nms_mask_kernel<<<div_up(static_cast<long long>(nms_pre_max_size) * 2 * cbmax * 32, 256), 256, 0, st>>>(at, w);
  P3D_LAUNCH_CHECK();
  ahp_greedy_kernel<<<1, 256, static_cast<size_t>(cbmax) * 8, st>>>(at, w);
  P3D_LAUNCH_CHECK();
  ahp_emit_kernel<<<1, 256, 0, st>>>(at, w, boxes, scores, reinterpret_cast<long long *>(labels), counts);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
