// centerpoint_postprocess for sm_90a: all tasks batched in every launch, no host synchronisation.
//
// Replaces paddle3d/ops/centerpoint_postprocess/postprocess.cu:104-280, which runs per task
// 4 Paddle elementwise ops + decode_kernel + 2 masked_select (D2H sync) + argsort + nms_kernel +
// blocking D2H of the bit-matrix + host greedy loop + cudaMemcpy H2D + 5 gathers (x6 tasks).
// Here:
//   P1 cpp_decode     sigmoid/max/argmax over the task's heat-map channels, box decode (exp, atan2f),
//                     threshold + raw-offset range test (the reference tests reg/height, NOT the decoded
//                     centre: postprocess.cu:72-77), candidates appended with warp-aggregated atomics
//                     as sortable 64-bit keys (~score_bits << 32 | cell).
//   P2 cpp_rank       exact descending-score order by rank counting (keys are unique; ties in score
//                     resolve to ascending cell index — this repo's defined argsort tie order);
//                     writes the first nms_pre_max_size cells in order.
//   P3 cpp_nms_mask   rotated-IoU suppression bit-matrix, upper triangle, boxes re-laid as
//                     (x, y, z, dim1, dim0, dim2, -rot - pi/2) exactly as
//                     centerpoint_postprocess/iou3d_nms_kernel.cu:299-307 (angle formed in double).
//   P4 cpp_greedy     on-device greedy reduction (nms_reduce.cuh), one CTA per task.
//   P5 cpp_emit       prefix over tasks, gathers, label offset, fake row for empty tasks
//                     (postprocess.cu:190-202), concatenated outputs + counts.
#include "box_geom.cuh"
#include "common.cuh"
#include "nms_reduce.cuh"

namespace p3d {
namespace {

constexpr int kMaxTasks = 16;

struct CppTasks {
  const float *hm[kMaxTasks];
  const float *reg[kMaxTasks];
  const float *height[kMaxTasks];
  const float *dim[kMaxTasks];
  const float *vel[kMaxTasks];
  const float *rot[kMaxTasks];
  int hm_c[kMaxTasks];
  int label_off[kMaxTasks];
};

struct CppAttrs {
  float vs_x, vs_y, pc_x, pc_y;
  float r_xmin, r_ymin, r_zmin, r_xmax, r_ymax, r_zmax;
  float down_ratio, score_thr, iou_thr;
  int W, HW, T, dims, with_vel, pre_max, post_max, cbmax;
};

struct CppWs {
  int32_t *cnt;                 // [T] candidates per task
  int32_t *nkeep;               // [T] boxes kept by the greedy pass
  unsigned long long *keys;     // [T, HW]
  float *boxes;                 // [T, HW, dims] (only candidate rows are written)
  float *score;                 // [T, HW]
  int32_t *label;               // [T, HW]
  int32_t *order;               // [T, pre_max] cell index of the r-th best candidate
  unsigned long long *mask;     // [T, pre_max, cbmax]
  int32_t *keep;                // [T, pre_max]
  size_t bytes;
};

CppWs carve(void *p, int T, int HW, int pre_max) {
  CppWs w;
  Carver c(p);
  const int cbmax = (pre_max + 63) / 64;
  w.cnt = c.take<int32_t>(2 * kMaxTasks);
  w.nkeep = w.cnt + kMaxTasks;
  w.keys = c.take<unsigned long long>(static_cast<size_t>(T) * HW);
  w.boxes = c.take<float>(static_cast<size_t>(T) * HW * 9);
  w.score = c.take<float>(static_cast<size_t>(T) * HW);
  w.label = c.take<int32_t>(static_cast<size_t>(T) * HW);
  w.order = c.take<int32_t>(static_cast<size_t>(T) * pre_max);
  w.mask = c.take<unsigned long long>(static_cast<size_t>(T) * pre_max * cbmax);
  w.keep = c.take<int32_t>(static_cast<size_t>(T) * pre_max);
  w.bytes = c.off;
  return w;
}

__global__ void __launch_bounds__(256) cpp_decode_kernel(CppTasks tk, CppAttrs at, CppWs w) {
  const int t = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool cand = false;
  float best = 0.f;
  if (i < at.HW) {
    const int HW = at.HW;
    const float *hm = tk.hm[t];
    int bl = 0;
    const int C = tk.hm_c[t];
    for (int c = 0; c < C; ++c) {
      const float s = 1.0f / (1.0f + expf(-hm[static_cast<size_t>(c) * HW + i]));  // paddle sigmoid, fp32
      if (c == 0 || s > best) {  // argmax keeps the first maximal channel
        best = s;
        bl = c;
      }
    }
    const float x = tk.reg[t][i], y = tk.reg[t][i + HW], z = tk.height[t][i];
    cand = best > at.score_thr && x <= at.r_xmax && y <= at.r_ymax && z <= at.r_zmax && x >= at.r_xmin &&
           y >= at.r_ymin && z >= at.r_zmin;
    if (cand) {
      const int xs = i % at.W, ys = i / at.W;
      float *b = w.boxes + (static_cast<size_t>(t) * HW + i) * at.dims;
      b[0] = (x + xs) * at.down_ratio * at.vs_x + at.pc_x;
      b[1] = (y + ys) * at.down_ratio * at.vs_y + at.pc_y;
      b[2] = z;
      b[3] = expf(tk.dim[t][i]);
      b[4] = expf(tk.dim[t][i + HW]);
      b[5] = expf(tk.dim[t][i + 2 * HW]);
      const float ang = atan2f(tk.rot[t][i], tk.rot[t][i + HW]);
      if (at.with_vel) {
        b[6] = tk.vel[t][i];
        b[7] = tk.vel[t][i + HW];
        b[8] = ang;
      } else {
        b[6] = ang;
      }
      w.score[static_cast<size_t>(t) * HW + i] = best;
      w.label[static_cast<size_t>(t) * HW + i] = bl;
    }
  }
  // warp-aggregated append
  const unsigned m = __ballot_sync(0xffffffffu, cand);
  if (m) {
    const int lane = threadIdx.x & 31;
    int base = 0;
    if (lane == __ffs(m) - 1) base = atomicAdd(&w.cnt[t], __popc(m));
    base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
    if (cand) {
      const unsigned long long key =
          (static_cast<unsigned long long>(~__float_as_uint(best)) << 32) | static_cast<unsigned int>(i);
      w.keys[static_cast<size_t>(t) * at.HW + base + __popc(m & ((1u << lane) - 1))] = key;
    }
  }
}

__global__ void __launch_bounds__(256) cpp_rank_kernel(CppAttrs at, CppWs w) {
  const int t = blockIdx.y;
  const int M = w.cnt[t];
  if (static_cast<int>(blockIdx.x * blockDim.x) >= M) return;
  __shared__ unsigned long long tile[256];
  const unsigned long long *keys = w.keys + static_cast<size_t>(t) * at.HW;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long mine = j < M ? keys[j] : ~0ull;
  int rank = 0;
  for (int k0 = 0; k0 < M; k0 += 256) {
    __syncthreads();
    tile[threadIdx.x] = (k0 + threadIdx.x < M) ? keys[k0 + threadIdx.x] : ~0ull;
    __syncthreads();
    const int lim = min(256, M - k0);
#pragma unroll 8
    for (int k = 0; k < lim; ++k) rank += (tile[k] < mine);
  }
  if (j < M && rank < at.pre_max) w.order[static_cast<size_t>(t) * at.pre_max + rank] = static_cast<int>(mine & 0xffffffffu);
}

__device__ __forceinline__ void fetch_nms_box(const float *b, int dims, float *o) {
  o[0] = b[0];
  o[1] = b[1];
  o[2] = b[2];
  o[3] = b[4];
  o[4] = b[3];
  o[5] = b[5];
  o[6] = -b[dims - 1] - 3.141592653589793 / 2;  // double arithmetic, rounded on store (reference :305-307)
}

__global__ void __launch_bounds__(64) cpp_nms_mask_kernel(CppAttrs at, CppWs w) {
  const int t = blockIdx.z, rb = blockIdx.y, cb = blockIdx.x;
  if (cb < rb) return;
  const int n = min(w.cnt[t], at.pre_max);
  if (rb * 64 >= n || cb * 64 >= n) return;
  const int rows = min(n - rb * 64, 64), cols = min(n - cb * 64, 64);
  const float *boxes = w.boxes + static_cast<size_t>(t) * at.HW * at.dims;
  const int32_t *order = w.order + static_cast<size_t>(t) * at.pre_max;
  __shared__ float s_col[64 * 7], s_row[64 * 7];
  __shared__ unsigned short s_pairs[64 * 64];
  __shared__ unsigned long long s_bits[64];
  __shared__ int s_cnt[3];
  if (threadIdx.x < cols)
    fetch_nms_box(boxes + static_cast<size_t>(order[cb * 64 + threadIdx.x]) * at.dims, at.dims, s_col + threadIdx.x * 7);
  if (threadIdx.x < rows)
    fetch_nms_box(boxes + static_cast<size_t>(order[rb * 64 + threadIdx.x]) * at.dims, at.dims, s_row + threadIdx.x * 7);
  __syncthreads();
  const unsigned long long bits = nms_rotated_tile(s_row, s_col, rows, cols, rb == cb, at.iou_thr, s_pairs, s_bits, s_cnt);
  if (threadIdx.x < rows) w.mask[(static_cast<size_t>(t) * at.pre_max + rb * 64 + threadIdx.x) * at.cbmax + cb] = bits;
}

__global__ void __launch_bounds__(256) cpp_greedy_kernel(CppAttrs at, CppWs w) {
  extern __shared__ unsigned long long s_dyn[];
  __shared__ unsigned long long s_misc[2];
  const int t = blockIdx.x;
  const int n = min(w.cnt[t], at.pre_max);
  const int k = nms_greedy_cta(w.mask + static_cast<size_t>(t) * at.pre_max * at.cbmax, n, at.cbmax,
                               w.keep + static_cast<size_t>(t) * at.pre_max, s_dyn, s_misc, at.post_max);
  if (threadIdx.x == 0) w.nkeep[t] = k;
}

__global__ void __launch_bounds__(256) cpp_emit_kernel(CppTasks tk, CppAttrs at, CppWs w, float *__restrict__ bboxes,
                                                       float *__restrict__ scores, long long *__restrict__ labels,
                                                       int32_t *__restrict__ counts) {
  __shared__ int s_rows[kMaxTasks], s_off[kMaxTasks + 1];
  if (threadIdx.x < at.T) {
    const int t = threadIdx.x;
    s_rows[t] = (w.cnt[t] == 0) ? 1 : min(w.nkeep[t], at.post_max);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int t = 0; t < at.T; ++t) {
      s_off[t] = acc;
      acc += s_rows[t];
      counts[t] = s_rows[t];
    }
    s_off[at.T] = acc;
    counts[at.T] = acc;
  }
  __syncthreads();
  const int total = s_off[at.T];
  for (int r = threadIdx.x; r < total; r += blockDim.x) {
    int t = 0;
    while (r >= s_off[t + 1]) ++t;
    const int rr = r - s_off[t];
    float *ob = bboxes + static_cast<size_t>(r) * at.dims;
    if (w.cnt[t] == 0) {
      for (int d = 0; d < at.dims; ++d) ob[d] = 0.f;
      scores[r] = -1.f;
      labels[r] = 0;
    } else {
      const int cell = w.order[static_cast<size_t>(t) * at.pre_max + w.keep[static_cast<size_t>(t) * at.pre_max + rr]];
      const float *b = w.boxes + (static_cast<size_t>(t) * at.HW + cell) * at.dims;
      for (int d = 0; d < at.dims; ++d) ob[d] = b[d];
      scores[r] = w.score[static_cast<size_t>(t) * at.HW + cell];
      labels[r] = static_cast<long long>(w.label[static_cast<size_t>(t) * at.HW + cell]) + tk.label_off[t];
    }
  }
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" size_t p3d_centerpoint_postprocess_workspace_bytes(int num_tasks, int feat_h, int feat_w,
                                                               int nms_pre_max_size, int nms_post_max_size) {
  (void)nms_post_max_size;
  if (num_tasks < 1 || num_tasks > kMaxTasks || feat_h < 1 || feat_w < 1 || nms_pre_max_size < 1) return 0;
  return carve(nullptr, num_tasks, feat_h * feat_w, nms_pre_max_size).bytes;
}

extern "C" int p3d_centerpoint_postprocess(int num_tasks, const float *const *hm, const int32_t *hm_channels_host,
                                           const float *const *reg, const float *const *height,
                                           const float *const *dim, const float *const *vel,
                                           const float *const *rot, int feat_h, int feat_w,
                                           const float *voxel_size_host, const float *point_cloud_range_host,
                                           const float *post_center_range_host, const int32_t *num_classes_host,
                                           int down_ratio, float score_threshold, float nms_iou_threshold,
                                           int nms_pre_max_size, int nms_post_max_size, int with_velocity,
                                           float *bboxes, float *scores, int64_t *labels, int32_t *counts,
                                           void *workspace, size_t workspace_bytes, p3d_stream_t stream) {
  if (num_tasks < 1 || num_tasks > kMaxTasks) return num_tasks < 1 ? P3D_ERR_INVALID_ARG : P3D_ERR_UNSUPPORTED;
  if (!hm || !hm_channels_host || !reg || !height || !dim || !vel || !rot || !voxel_size_host ||
      !point_cloud_range_host || !post_center_range_host || !num_classes_host || !bboxes || !scores || !labels ||
      !counts || !workspace || feat_h < 1 || feat_w < 1 || nms_pre_max_size < 1 || nms_post_max_size < 0)
    return P3D_ERR_INVALID_ARG;
  const int HW = feat_h * feat_w;
  CppWs w = carve(workspace, num_tasks, HW, nms_pre_max_size);
  if (workspace_bytes < w.bytes) return P3D_ERR_WORKSPACE;
  CppTasks tk;
  for (int t = 0; t < num_tasks; ++t) {
    if (!hm[t] || !reg[t] || !height[t] || !dim[t] || !vel[t] || !rot[t] || hm_channels_host[t] < 1)
      return P3D_ERR_INVALID_ARG;
    tk.hm[t] = hm[t];
    tk.reg[t] = reg[t];
    tk.height[t] = height[t];
    tk.dim[t] = dim[t];
    tk.vel[t] = vel[t];
    tk.rot[t] = rot[t];
    tk.hm_c[t] = hm_channels_host[t];
    tk.label_off[t] = num_classes_host[t];
  }
  CppAttrs at;
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
  at.down_ratio = static_cast<float>(down_ratio);
  at.score_thr = score_threshold;
  at.iou_thr = nms_iou_threshold;
  at.W = feat_w;
  at.HW = HW;
  at.T = num_tasks;
  at.dims = with_velocity ? 9 : 7;
  at.with_vel = with_velocity ? 1 : 0;
  at.pre_max = nms_pre_max_size;
  at.post_max = nms_post_max_size;
  at.cbmax = (nms_pre_max_size + 63) / 64;
  if (static_cast<size_t>(at.cbmax) * 8 > 48 * 1024) return P3D_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  P3D_CUDA_CHECK(cudaMemsetAsync(w.cnt, 0, sizeof(int32_t) * 2 * kMaxTasks, st));
  dim3 g1(div_up(HW, 256), num_tasks);
  cpp_decode_kernel<<<g1, 256, 0, st>>>(tk, at, w);
  P3D_LAUNCH_CHECK();
  cpp_rank_kernel<<<g1, 256, 0, st>>>(at, w);
  P3D_LAUNCH_CHECK();
  dim3 g3(at.cbmax, at.cbmax, num_tasks);
  cpp_nms_mask_kernel<<<g3, 64, 0, st>>>(at, w);
  P3D_LAUNCH_CHECK();
  cpp_greedy_kernel<<<num_tasks, 256, static_cast<size_t>(at.cbmax) * 8, st>>>(at, w);
  P3D_LAUNCH_CHECK();
  cpp_emit_kernel<<<1, 256, 0, st>>>(tk, at, w, bboxes, scores, reinterpret_cast<long long *>(labels), counts);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
