// bevdet_postprocess for sm_90a: BEVDet's CenterHead.get_bboxes (CenterPointBBoxCoder.decode + get_task_detections with
// per-class scale-NMS or circle NMS) for all tasks in every launch, no host synchronisation, no allocation.
// PARITY UNPINNED: the semantics are recalled from BEVDet's head, from which Paddle3D's configs/bevdet head descends
// (include/p3d_b200.h states them).  It differs from centerpoint_postprocess (postprocess.cu) in every rule, so the two
// share box_geom.cuh / nms_reduce.cuh and nothing else:
//   B1 bdp_candidates  one pass over every heat-map value of every task: sigmoid, score > threshold, (class, cell)
//                      candidates appended with warp-aggregated atomics as sortable 64-bit keys
//                      (~score_bits << 32 | class * HW + cell).  Only the heat maps are read here.
//   B2 bdp_select      one CTA per task: the max_num smallest keys in exact order (topk_select.cuh: radix select,
//                      then a rank count of the keys at or below the cut).  Keys are unique, so equal scores order by
//                      ascending class * HW + cell.
//   B3 bdp_decode      box decode of the selected candidates, range test on the DECODED centre (a box with a non-finite
//                      value is dropped as well), survivors compacted in score order with a block-wide scan.
//   B4 bdp_mask        upper triangle of the suppression bit-matrix in 64 x 64 tiles: rotated IoU on boxes whose dx, dy
//                      were scaled by the class's nms_rescale_factor when the tile was loaded, or the squared centre
//                      distance against min_radius for a circle task.
//   B5 bdp_greedy      on-device greedy reduction (nms_reduce.cuh), one CTA per task, stops at post_max_size.
//   B6 bdp_emit        prefix over tasks, gather, z to the bottom centre, label offset, counts.  No row for an empty task.
#include "box_geom.cuh"
#include "common.cuh"
#include "nms_reduce.cuh"
#include "topk_select.cuh"

namespace p3d {
namespace {

constexpr int kMaxTasks = 16;
constexpr int kMaxClasses = 64;  // over all tasks
constexpr int kBoxDims = 9;      // x, y, z, dx, dy, dz, rot, vx, vy

struct BdpTasks {
  const float *hm[kMaxTasks];
  const float *reg[kMaxTasks];
  const float *height[kMaxTasks];
  const float *dim[kMaxTasks];
  const float *vel[kMaxTasks];
  const float *rot[kMaxTasks];
  int hm_c[kMaxTasks];
  int key_off[kMaxTasks];   // first key of the task: sum of hm_c * HW of the tasks before it
  int low_bits[kMaxTasks];  // bits of hm_c * HW - 1: the key's digits from there up to bit 32 are zero
  int label_off[kMaxTasks];
};

// per-task suppression rule
struct BdpNms {
  int type[kMaxTasks];
  float thr[kMaxTasks];
  float radius[kMaxTasks];
  int cls_off[kMaxTasks];
  float rescale[kMaxClasses];  // one factor per class, tasks concatenated
};

struct BdpAttrs {
  float vs_x, vs_y, pc_x, pc_y;
  float r_xmin, r_ymin, r_zmin, r_xmax, r_ymax, r_zmax;
  float out_size_factor, score_thr;
  int W, HW, T, cmax, max_num, pre_max, post_max, cbmax;
};

struct BdpWs {
  int32_t *cnt;              // [T] candidates per task
  int32_t *nsel;             // [T] min(candidates, max_num)
  int32_t *nvalid;           // [T] selected candidates inside the range
  int32_t *nkeep;            // [T] boxes kept by the greedy pass
  unsigned long long *keys;  // [sum hm_c * HW]
  unsigned long long *sel;   // [T, max_num] the keys at or below the cut, unordered
  unsigned long long *sorted;  // [T, max_num] the same keys in order
  float *boxes;              // [T, max_num, 9] survivors of the range test, in score order (z = gravity centre)
  float *score;              // [T, max_num]
  int32_t *cls;              // [T, max_num]
  unsigned long long *mask;  // [T, max_num, cbmax]
  int32_t *keep;             // [T, max_num]
  size_t bytes;
};

BdpWs carve(void *p, int T, size_t total_keys, int max_num) {
  BdpWs w;
  Carver c(p);
  const size_t n = static_cast<size_t>(T) * max_num;
  const int cbmax = (max_num + 63) / 64;
  w.cnt = c.take<int32_t>(4 * kMaxTasks);
  w.nsel = w.cnt + kMaxTasks;
  w.nvalid = w.cnt + 2 * kMaxTasks;
  w.nkeep = w.cnt + 3 * kMaxTasks;
  w.keys = c.take<unsigned long long>(total_keys);
  w.sel = c.take<unsigned long long>(n);
  w.sorted = c.take<unsigned long long>(n);
  w.boxes = c.take<float>(n * kBoxDims);
  w.score = c.take<float>(n);
  w.cls = c.take<int32_t>(n);
  w.mask = c.take<unsigned long long>(n * cbmax);
  w.keep = c.take<int32_t>(n);
  w.bytes = c.off;
  return w;
}

__global__ void __launch_bounds__(256) bdp_candidates_kernel(BdpTasks tk, BdpAttrs at, BdpWs w) {
  const int t = blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;  // class * HW + cell
  bool cand = false;
  float s = 0.f;
  if (j < tk.hm_c[t] * at.HW) {
    s = 1.0f / (1.0f + expf(-tk.hm[t][j]));  // as cpp_decode_kernel
    cand = s > at.score_thr;                 // false for a NaN logit
  }
  const unsigned m = __ballot_sync(0xffffffffu, cand);
  if (m) {
    const int lane = threadIdx.x & 31;
    int base = 0;
    if (lane == __ffs(m) - 1) base = atomicAdd(&w.cnt[t], __popc(m));
    base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
    if (cand)
      w.keys[tk.key_off[t] + base + __popc(m & ((1u << lane) - 1))] =
          (static_cast<unsigned long long>(~__float_as_uint(s)) << 32) | static_cast<unsigned int>(j);
  }
}

__global__ void __launch_bounds__(1024) bdp_select_kernel(BdpTasks tk, BdpAttrs at, BdpWs w) {
  const int t = blockIdx.x;
  const size_t o = static_cast<size_t>(t) * at.max_num;
  const int K = select_smallest_keys(w.keys + tk.key_off[t], w.cnt[t], at.max_num, tk.low_bits[t], w.sel + o,
                                     w.sorted + o);
  if (threadIdx.x == 0) w.nsel[t] = K;
}

__global__ void __launch_bounds__(256) bdp_decode_kernel(BdpTasks tk, BdpAttrs at, BdpWs w) {
  const int t = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int K = w.nsel[t], HW = at.HW;
  const unsigned long long *sorted = w.sorted + static_cast<size_t>(t) * at.max_num;
  __shared__ int s_w[8];
  int total = 0;
  for (int r0 = 0; r0 < K; r0 += 256) {
    const int r = r0 + tid;
    bool ok = false;
    float b[kBoxDims], s = 0.f;
    int c = 0;
    if (r < K) {
      const unsigned long long key = sorted[r];
      s = __uint_as_float(~static_cast<unsigned int>(key >> 32));
      const int j = static_cast<int>(key & 0xffffffffu);
      c = j / HW;
      const int i = j - c * HW;
      const int xs = i % at.W, ys = i / at.W;
      // cpp_decode_kernel's expressions, every operation rounded on its own (no fused multiply-add)
      b[0] = __fadd_rn(__fmul_rn(__fmul_rn(__fadd_rn(tk.reg[t][i], static_cast<float>(xs)), at.out_size_factor), at.vs_x), at.pc_x);
      b[1] = __fadd_rn(__fmul_rn(__fmul_rn(__fadd_rn(tk.reg[t][i + HW], static_cast<float>(ys)), at.out_size_factor), at.vs_y), at.pc_y);
      b[2] = tk.height[t][i];
      // the range test is false for a NaN centre
      ok = b[0] >= at.r_xmin && b[0] <= at.r_xmax && b[1] >= at.r_ymin && b[1] <= at.r_ymax && b[2] >= at.r_zmin &&
           b[2] <= at.r_zmax;
      if (ok) {
        b[3] = expf(tk.dim[t][i]);
        b[4] = expf(tk.dim[t][i + HW]);
        b[5] = expf(tk.dim[t][i + 2 * HW]);
        b[6] = atan2f(tk.rot[t][i], tk.rot[t][i + HW]);
        b[7] = tk.vel[t][i];
        b[8] = tk.vel[t][i + HW];
        // a box with a NaN or infinite value is dropped: every row emitted is finite, and the suppression stage never
        // sees a box its geometry was not written for
#pragma unroll
        for (int d = 3; d < kBoxDims; ++d) ok = ok && isfinite(b[d]);
      }
    }
    // order-preserving compaction: ballot within the warp, the 8 warp counts through shared memory
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_w[wid] = __popc(m);
    __syncthreads();
    int before = 0, round = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      before += q < wid ? s_w[q] : 0;
      round += s_w[q];
    }
    if (ok) {
      const size_t o = static_cast<size_t>(t) * at.max_num + total + before + __popc(m & ((1u << lane) - 1));
#pragma unroll
      for (int d = 0; d < kBoxDims; ++d) w.boxes[o * kBoxDims + d] = b[d];
      w.score[o] = s;
      w.cls[o] = c;
    }
    total += round;
    __syncthreads();
  }
  if (tid == 0) w.nvalid[t] = total;
}

__global__ void __launch_bounds__(64) bdp_mask_kernel(BdpAttrs at, BdpNms nm, BdpWs w) {
  const int t = blockIdx.z, rb = blockIdx.y, cb = blockIdx.x;
  if (cb < rb) return;
  const int n = min(w.nvalid[t], at.pre_max);
  if (rb * 64 >= n || cb * 64 >= n) return;
  const int rows = min(n - rb * 64, 64), cols = min(n - cb * 64, 64);
  __shared__ float s_col[64 * 7], s_row[64 * 7];
  __shared__ unsigned short s_pairs[64 * 64];
  __shared__ unsigned long long s_bits[64];
  __shared__ int s_cnt[3];
  const int tid = threadIdx.x;
  // (x, y, z, dx * f, dy * f, dz, rot) with f the rescale factor of the box's class
  auto fetch = [&](int idx, float *o) {
    const size_t r = static_cast<size_t>(t) * at.max_num + idx;
    const float *b = w.boxes + r * kBoxDims;
    const float f = nm.rescale[nm.cls_off[t] + w.cls[r]];
    o[0] = b[0];
    o[1] = b[1];
    o[2] = b[2];
    o[3] = b[3] * f;
    o[4] = b[4] * f;
    o[5] = b[5];
    o[6] = b[6];
  };
  if (tid < cols) fetch(cb * 64 + tid, s_col + tid * 7);
  if (tid < rows) fetch(rb * 64 + tid, s_row + tid * 7);
  __syncthreads();
  unsigned long long bits = 0ull;
  if (nm.type[t] == P3D_BEVDET_NMS_ROTATE) {
    bits = nms_rotated_tile(s_row, s_col, rows, cols, rb == cb, nm.thr[t], s_pairs, s_bits, s_cnt);
  } else if (tid < rows) {  // circle_nms: squared centre distance against min_radius itself, fp32, no fused multiply-add
    const float x = s_row[tid * 7], y = s_row[tid * 7 + 1], rad = nm.radius[t];
    for (int j = rb == cb ? tid + 1 : 0; j < cols; ++j) {
      const float dx = x - s_col[j * 7], dy = y - s_col[j * 7 + 1];
      if (__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) <= rad) bits |= 1ull << j;
    }
  }
  if (tid < rows) w.mask[(static_cast<size_t>(t) * at.max_num + rb * 64 + tid) * at.cbmax + cb] = bits;
}

__global__ void __launch_bounds__(256) bdp_greedy_kernel(BdpAttrs at, BdpWs w) {
  extern __shared__ unsigned long long s_dyn[];
  __shared__ unsigned long long s_misc[2];
  const int t = blockIdx.x;
  const int n = min(w.nvalid[t], at.pre_max);
  const int k = nms_greedy_cta(w.mask + static_cast<size_t>(t) * at.max_num * at.cbmax, n, at.cbmax,
                               w.keep + static_cast<size_t>(t) * at.max_num, s_dyn, s_misc, at.post_max);
  if (threadIdx.x == 0) w.nkeep[t] = k;
}

__global__ void __launch_bounds__(256) bdp_emit_kernel(BdpTasks tk, BdpAttrs at, BdpWs w, float *__restrict__ bboxes,
                                                       float *__restrict__ scores, long long *__restrict__ labels,
                                                       int32_t *__restrict__ counts) {
  __shared__ int s_off[kMaxTasks + 1];
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int t = 0; t < at.T; ++t) {
      const int rows = min(w.nkeep[t], at.post_max);
      s_off[t] = acc;
      acc += rows;
      counts[t] = rows;
    }
    s_off[at.T] = acc;
    counts[at.T] = acc;
  }
  __syncthreads();
  const int total = s_off[at.T];
  for (int r = threadIdx.x; r < total; r += blockDim.x) {
    int t = 0;
    while (r >= s_off[t + 1]) ++t;
    const size_t src = static_cast<size_t>(t) * at.max_num + w.keep[static_cast<size_t>(t) * at.max_num + r - s_off[t]];
    const float *b = w.boxes + src * kBoxDims;
    float *ob = bboxes + static_cast<size_t>(r) * kBoxDims;
#pragma unroll
    for (int d = 0; d < kBoxDims; ++d) ob[d] = b[d];
    // dims are the decoded ones: the reference scales them by the factor for the NMS and divides again, which is this
    // value or its neighbour (at most one ulp away)
    ob[2] = b[2] - b[5] * 0.5f;  // bottom centre
    scores[r] = w.score[src];
    labels[r] = static_cast<long long>(w.cls[src]) + tk.label_off[t];
  }
}

bool sizes(int T, const int32_t *hm_c, int H, int W, int max_num, size_t *total_keys) {
  if (T < 1 || T > kMaxTasks || !hm_c || H < 1 || W < 1 || max_num < 1) return false;
  const long long HW = static_cast<long long>(H) * W;
  long long keys = 0, classes = 0;
  for (int t = 0; t < T; ++t) {
    if (hm_c[t] < 1) return false;
    classes += hm_c[t];
    keys += hm_c[t] * HW;
  }
  if (classes > kMaxClasses || keys > 0x7fffffffll) return false;
  *total_keys = static_cast<size_t>(keys);
  return true;
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" size_t p3d_bevdet_postprocess_workspace_bytes(int num_tasks, const int32_t *hm_channels_host, int feat_h,
                                                          int feat_w, int max_num) {
  size_t keys = 0;
  if (!sizes(num_tasks, hm_channels_host, feat_h, feat_w, max_num, &keys)) return 0;
  return carve(nullptr, num_tasks, keys, max_num).bytes;
}

extern "C" int p3d_bevdet_postprocess(int num_tasks, const float *const *hm, const int32_t *hm_channels_host,
                                      const float *const *reg, const float *const *height, const float *const *dim,
                                      const float *const *vel, const float *const *rot, int feat_h, int feat_w,
                                      const float *voxel_size_host, const float *point_cloud_range_host,
                                      const float *post_center_range_host, int out_size_factor, float score_threshold,
                                      int max_num, int pre_max_size, int post_max_size, const int32_t *nms_type_host,
                                      const float *nms_thr_host, const float *min_radius_host,
                                      const float *rescale_host, const int32_t *label_offset_host, float *bboxes,
                                      float *scores, int64_t *labels, int32_t *counts, void *workspace,
                                      size_t workspace_bytes, p3d_stream_t stream) {
  if (num_tasks < 1) return P3D_ERR_INVALID_ARG;
  if (num_tasks > kMaxTasks) return P3D_ERR_UNSUPPORTED;
  if (!hm || !hm_channels_host || !reg || !height || !dim || !vel || !rot || !voxel_size_host ||
      !point_cloud_range_host || !post_center_range_host || !nms_type_host || !nms_thr_host || !min_radius_host ||
      !rescale_host || !label_offset_host || !bboxes || !scores || !labels || !counts || feat_h < 1 || feat_w < 1 ||
      out_size_factor < 1 || max_num < 1 || pre_max_size < 1 || post_max_size < 1)
    return P3D_ERR_INVALID_ARG;
  const int T = num_tasks, HW = feat_h * feat_w;
  BdpTasks tk;
  BdpNms nm;
  int classes = 0;
  for (int t = 0; t < T; ++t) {
    if (hm_channels_host[t] < 1) return P3D_ERR_INVALID_ARG;
    classes += hm_channels_host[t];
  }
  size_t total_keys = 0;
  if (!sizes(T, hm_channels_host, feat_h, feat_w, max_num, &total_keys)) return P3D_ERR_UNSUPPORTED;
  int key_off = 0, cls_off = 0, cmax = 1;
  for (int t = 0; t < T; ++t) {
    const int C = hm_channels_host[t];
    if (!hm[t] || !reg[t] || !height[t] || !dim[t] || !vel[t] || !rot[t]) return P3D_ERR_INVALID_ARG;
    if (nms_type_host[t] != P3D_BEVDET_NMS_ROTATE && nms_type_host[t] != P3D_BEVDET_NMS_CIRCLE) return P3D_ERR_INVALID_ARG;
    if (!(min_radius_host[t] >= 0.f)) return P3D_ERR_INVALID_ARG;
    for (int c = 0; c < C; ++c) {
      if (!(rescale_host[cls_off + c] > 0.f)) return P3D_ERR_INVALID_ARG;
      nm.rescale[cls_off + c] = rescale_host[cls_off + c];
    }
    tk.hm[t] = hm[t];
    tk.reg[t] = reg[t];
    tk.height[t] = height[t];
    tk.dim[t] = dim[t];
    tk.vel[t] = vel[t];
    tk.rot[t] = rot[t];
    tk.hm_c[t] = C;
    tk.key_off[t] = key_off;
    tk.low_bits[t] = 1;
    while (tk.low_bits[t] < 32 && ((static_cast<long long>(C) * HW - 1) >> tk.low_bits[t])) ++tk.low_bits[t];
    tk.label_off[t] = label_offset_host[t];
    nm.type[t] = nms_type_host[t];
    nm.thr[t] = nms_thr_host[t];
    nm.radius[t] = min_radius_host[t];
    nm.cls_off[t] = cls_off;
    key_off += C * HW;
    cls_off += C;
    cmax = C > cmax ? C : cmax;
  }
  for (int c = classes; c < kMaxClasses; ++c) nm.rescale[c] = 1.f;
  BdpWs w = carve(workspace, T, total_keys, max_num);
  if (!workspace || workspace_bytes < w.bytes) return P3D_ERR_WORKSPACE;
  BdpAttrs at;
  at.vs_x = voxel_size_host[0];
  at.vs_y = voxel_size_host[1];
  at.pc_x = point_cloud_range_host[0];
  at.pc_y = point_cloud_range_host[1];
  at.r_xmin = post_center_range_host[0];
  at.r_ymin = post_center_range_host[1];
  at.r_zmin = post_center_range_host[2];
  at.r_xmax = post_center_range_host[3];
  at.r_ymax = post_center_range_host[4];
  at.r_zmax = post_center_range_host[5];
  at.out_size_factor = static_cast<float>(out_size_factor);
  at.score_thr = score_threshold;
  at.W = feat_w;
  at.HW = HW;
  at.T = T;
  at.cmax = cmax;
  at.max_num = max_num;
  at.pre_max = pre_max_size;
  at.post_max = post_max_size;
  at.cbmax = (max_num + 63) / 64;
  if (static_cast<size_t>(at.cbmax) * 8 > 48 * 1024) return P3D_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  P3D_CUDA_CHECK(cudaMemsetAsync(w.cnt, 0, sizeof(int32_t) * 4 * kMaxTasks, st));
  bdp_candidates_kernel<<<dim3(div_up(static_cast<long long>(cmax) * HW, 256), T), 256, 0, st>>>(tk, at, w);
  P3D_LAUNCH_CHECK();
  bdp_select_kernel<<<T, 1024, 0, st>>>(tk, at, w);
  P3D_LAUNCH_CHECK();
  bdp_decode_kernel<<<T, 256, 0, st>>>(tk, at, w);
  P3D_LAUNCH_CHECK();
  const int cb = (min(max_num, pre_max_size) + 63) / 64;  // tiles that can hold a box
  bdp_mask_kernel<<<dim3(cb, cb, T), 64, 0, st>>>(at, nm, w);
  P3D_LAUNCH_CHECK();
  bdp_greedy_kernel<<<T, 256, static_cast<size_t>(at.cbmax) * 8, st>>>(at, w);
  P3D_LAUNCH_CHECK();
  bdp_emit_kernel<<<1, 256, 0, st>>>(tk, at, w, bboxes, scores, reinterpret_cast<long long *>(labels), counts);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
