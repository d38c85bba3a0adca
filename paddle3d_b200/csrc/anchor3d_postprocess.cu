// anchor3d_postprocess for sm_90a: mmdet3d's Anchor3DHead.get_bboxes_single + box3d_multiclass_nms (BEVFusion's head)
// at batch 1 for every class in one set of launches, no host synchronisation, no allocation.  PARITY UNPINNED:
// include/p3d_b200.h states the six rules; tests/bevfusion_oracle.py restates them in numpy.  It differs from the SECOND
// anchor postprocess (anchor_postprocess.cu: class-agnostic NMS, area mask, score >= thr) in every rule, so the two share
// box_geom.cuh / nms_reduce.cuh and nothing else; the top-K is topk_select.cuh, shared with bevdet_postprocess.cu.
//   N1 a3d_score    per anchor: max over the classes of sigmoid(cls) (NaN if a class is NaN).  An anchor that can reach
//                   the output (a class score > score_thr, or a NaN score) appends its key with warp-aggregated atomics:
//                   (~score_bits << 32 | anchor) when A > nms_pre (descending score, ties by the lower anchor index, a
//                   NaN score first: key 0 above every number), the anchor index alone otherwise (anchor order).
//                   The others cannot enter the output and rank below every anchor that can, so leaving them out of
//                   the ranking changes no kept anchor and no kept order.
//   N2 a3d_select   one CTA: the nms_pre smallest keys in order -> the kept anchors in kept order.
//   N3 a3d_decode   per kept anchor: DeltaXYZWLHRBBoxCoder.decode and the dir label; a box with a non-finite value is
//                   dropped (the suppression geometry is not written for one); for every class with sigmoid(cls_c) >
//                   score_thr a key (~score_c_bits << 32 | kept position) is appended to the class's list.
//   N4 a3d_sort     one CTA per class: rank count of the class's keys -> descending class score, ties by kept order.
//   N5 a3d_mask     upper triangle of each class's suppression bit-matrix in 64 x 64 tiles (nms_rotated_tile) on
//                   (x, y, z, w, l, h, r) as (x, y, z, dx, dy, dz, heading).
//   N6 a3d_greedy   on-device greedy reduction (nms_reduce.cuh), one CTA per class, stops at max_num kept.
//   N7 a3d_concat   the classes' survivors concatenated in class order with (~score_bits << 32 | position) keys.
//   N8 a3d_emit     above max_num rows: each row's rank by counting smaller keys (score descending, ties in class-major
//                   order), rows ranked below max_num written; otherwise rows in class-major order.  Direction fix.
// A class keeps at most max_num rows: its later rows have max_num rows of the same class before them in the score sort,
// so they never reach the output, and the total still exceeds max_num exactly when the uncut total does or equals it.
// The fp32 expressions of N3 / N8 are written with explicit roundings (no fused multiply-add) so that the numpy
// restatement computes the same values.
#include "box_geom.cuh"
#include "common.cuh"
#include "nms_reduce.cuh"
#include "topk_select.cuh"

namespace p3d {
namespace {

constexpr int kMaxClasses = 64;
constexpr int kMaxPre = 4096;
constexpr int kCode = 9;  // x, y, z, w, l, h, r, vx, vy
constexpr float kPi = 3.14159274f;  // fp32(pi), as torch rounds np.pi against an fp32 tensor

struct A3dAttrs {
  int A, HW, R, C, pre, max_num, cbmax, low_bits, cap;  // cap = min(pre, max_num): rows per class after the greedy cut
  float score_thr, nms_thr, dir_off, dir_lim;
};

struct A3dWs {
  int32_t *cnt;              // [0] candidates, [1] kept anchors, [2, 2 + C) class list sizes, [2 + C, 2 + 2C) kept
  unsigned long long *keys;  // [A]
  unsigned long long *sel;   // [pre]
  unsigned long long *sorted;  // [pre]
  float *boxes;              // [pre, 9] decoded kept anchors
  int32_t *dir;              // [pre]
  unsigned long long *ckeys;   // [C, pre] class lists, unordered
  unsigned long long *csel;    // [C, pre] scratch of the sort
  unsigned long long *csorted; // [C, pre] the same in order
  unsigned long long *mask;  // [C, pre, cbmax]
  int32_t *keep;             // [C, pre]
  unsigned long long *flat;  // [C * cap] concatenated survivors
  size_t bytes;
};

A3dWs carve(void *p, long long A, int C, int pre, int max_num) {
  A3dWs w;
  Carver c(p);
  const size_t n = static_cast<size_t>(C) * pre;
  const int cbmax = (pre + 63) / 64;
  w.cnt = c.take<int32_t>(2 + 2 * kMaxClasses);
  w.keys = c.take<unsigned long long>(static_cast<size_t>(A));
  w.sel = c.take<unsigned long long>(pre);
  w.sorted = c.take<unsigned long long>(pre);
  w.boxes = c.take<float>(static_cast<size_t>(pre) * kCode);
  w.dir = c.take<int32_t>(pre);
  w.ckeys = c.take<unsigned long long>(n);
  w.csel = c.take<unsigned long long>(n);
  w.csorted = c.take<unsigned long long>(n);
  w.mask = c.take<unsigned long long>(n * cbmax);
  w.keep = c.take<int32_t>(n);
  w.flat = c.take<unsigned long long>(static_cast<size_t>(C) * (pre < max_num ? pre : max_num));
  w.bytes = c.off;
  return w;
}

__device__ __forceinline__ float sigmoid_f32(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }

__global__ void __launch_bounds__(256) a3d_score_kernel(const float *__restrict__ head, A3dAttrs at, A3dWs w) {
  // consecutive threads take consecutive cells of one anchor slot a, so each class plane is read coalesced
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  bool cand = false;
  unsigned long long key = 0ull;
  if (t < at.A) {
    const int a = t / at.HW, cell = t - a * at.HW;
    const int i = cell * at.R + a;
    const float *cls = head + static_cast<size_t>(a) * at.C * at.HW + cell;
    float best = sigmoid_f32(cls[0]);
    for (int c = 1; c < at.C && best == best; ++c) {
      const float s = sigmoid_f32(cls[static_cast<size_t>(c) * at.HW]);
      if (s > best || s != s) best = s;
    }
    cand = best != best || best > at.score_thr;
    const unsigned hi = best != best ? 0u : ~__float_as_uint(best);
    key = at.A > at.pre ? (static_cast<unsigned long long>(hi) << 32) | static_cast<unsigned>(i) : static_cast<unsigned>(i);
  }
  const unsigned m = __ballot_sync(0xffffffffu, cand);
  if (m) {
    const int lane = threadIdx.x & 31;
    int base = 0;
    if (lane == __ffs(m) - 1) base = atomicAdd(&w.cnt[0], __popc(m));
    base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
    if (cand) w.keys[base + __popc(m & ((1u << lane) - 1))] = key;
  }
}

__global__ void __launch_bounds__(1024) a3d_select_kernel(A3dAttrs at, A3dWs w) {
  const int K = select_smallest_keys(w.keys, w.cnt[0], at.pre, at.low_bits, w.sel, w.sorted);
  if (threadIdx.x == 0) w.cnt[1] = K;
}

__global__ void __launch_bounds__(128) a3d_decode_kernel(const float *__restrict__ head, const float *__restrict__ anchors,
                                                         A3dAttrs at, A3dWs w) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= w.cnt[1]) return;
  const int i = static_cast<int>(w.sorted[r] & 0xffffffffull);
  const int cell = i / at.R, a = i - cell * at.R;
  const size_t HW = at.HW;
  const float *an = anchors + static_cast<size_t>(i) * kCode;
  const float xa = an[0], ya = an[1], wa = an[3], la = an[4], ha = an[5], ra = an[6];
  const float *bt = head + (static_cast<size_t>(at.R) * at.C + a * kCode) * HW + cell;
  const float za = __fadd_rn(an[2], __fmul_rn(ha, 0.5f));
  const float diag = __fsqrt_rn(__fadd_rn(__fmul_rn(la, la), __fmul_rn(wa, wa)));
  float b[kCode];
  b[0] = __fadd_rn(__fmul_rn(bt[0], diag), xa);
  b[1] = __fadd_rn(__fmul_rn(bt[HW], diag), ya);
  const float zg = __fadd_rn(__fmul_rn(bt[2 * HW], ha), za);
  b[3] = __fmul_rn(expf(bt[3 * HW]), wa);
  b[4] = __fmul_rn(expf(bt[4 * HW]), la);
  b[5] = __fmul_rn(expf(bt[5 * HW]), ha);
  b[6] = __fadd_rn(bt[6 * HW], ra);
  b[2] = __fsub_rn(zg, __fmul_rn(b[5], 0.5f));
  b[7] = __fadd_rn(bt[7 * HW], an[7]);
  b[8] = __fadd_rn(bt[8 * HW], an[8]);
  const float *dt = head + (static_cast<size_t>(at.R) * (at.C + kCode) + a * 2) * HW + cell;
  w.dir[r] = dt[HW] > dt[0] ? 1 : 0;  // argmax, a tie to bin 0
  bool ok = true;
#pragma unroll
  for (int k = 0; k < kCode; ++k) {
    w.boxes[static_cast<size_t>(r) * kCode + k] = b[k];
    ok = ok && isfinite(b[k]);
  }
  if (!ok) return;
  const float *cls = head + static_cast<size_t>(a) * at.C * HW + cell;
  for (int c = 0; c < at.C; ++c) {
    const float s = sigmoid_f32(cls[c * HW]);
    if (s > at.score_thr)  // false for NaN
      w.ckeys[static_cast<size_t>(c) * at.pre + atomicAdd(&w.cnt[2 + c], 1)] =
          (static_cast<unsigned long long>(~__float_as_uint(s)) << 32) | static_cast<unsigned>(r);
  }
}

__global__ void __launch_bounds__(1024) a3d_sort_kernel(A3dAttrs at, A3dWs w) {
  const int c = blockIdx.x;
  const size_t o = static_cast<size_t>(c) * at.pre;
  select_smallest_keys(w.ckeys + o, w.cnt[2 + c], at.pre, 32, w.csel + o, w.csorted + o);
}

__global__ void __launch_bounds__(64) a3d_mask_kernel(A3dAttrs at, A3dWs w) {
  const int c = blockIdx.z, rb = blockIdx.y, cb = blockIdx.x;
  if (cb < rb) return;
  const int n = w.cnt[2 + c];
  if (rb * 64 >= n || cb * 64 >= n) return;
  const int rows = min(n - rb * 64, 64), cols = min(n - cb * 64, 64);
  __shared__ float s_col[64 * 7], s_row[64 * 7];
  __shared__ unsigned short s_pairs[64 * 64];
  __shared__ unsigned long long s_bits[64];
  __shared__ int s_cnt[3];
  const int tid = threadIdx.x;
  const unsigned long long *cs = w.csorted + static_cast<size_t>(c) * at.pre;
  auto fetch = [&](int idx, float *o) {
    const float *b = w.boxes + (cs[idx] & 0xffffffffull) * kCode;
#pragma unroll
    for (int k = 0; k < 7; ++k) o[k] = b[k];
  };
  if (tid < cols) fetch(cb * 64 + tid, s_col + tid * 7);
  if (tid < rows) fetch(rb * 64 + tid, s_row + tid * 7);
  __syncthreads();
  const unsigned long long bits = nms_rotated_tile(s_row, s_col, rows, cols, rb == cb, at.nms_thr, s_pairs, s_bits, s_cnt);
  if (tid < rows) w.mask[(static_cast<size_t>(c) * at.pre + rb * 64 + tid) * at.cbmax + cb] = bits;
}

__global__ void __launch_bounds__(256) a3d_greedy_kernel(A3dAttrs at, A3dWs w) {
  extern __shared__ unsigned long long s_dyn[];
  __shared__ unsigned long long s_misc[2];
  const int c = blockIdx.x;
  const int k = nms_greedy_cta(w.mask + static_cast<size_t>(c) * at.pre * at.cbmax, w.cnt[2 + c], at.cbmax,
                               w.keep + static_cast<size_t>(c) * at.pre, s_dyn, s_misc, at.max_num);
  if (threadIdx.x == 0) w.cnt[2 + at.C + c] = min(k, at.max_num);
}

// Rows before class c and the total, from the per-class kept counts.
__device__ __forceinline__ int class_offset(const A3dAttrs &at, const int32_t *kept, int c, int *total) {
  int off = 0, t = 0;
  for (int k = 0; k < at.C; ++k) {
    off += k < c ? kept[k] : 0;
    t += kept[k];
  }
  *total = t;
  return off;
}

// thread (c, j): survivor j of class c
__global__ void __launch_bounds__(256) a3d_concat_kernel(A3dAttrs at, A3dWs w) {
  const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int c = static_cast<int>(t / at.cap), j = static_cast<int>(t - static_cast<long long>(c) * at.cap);
  if (c >= at.C) return;
  const int32_t *kept = w.cnt + 2 + at.C;
  if (j >= kept[c]) return;
  int total;
  const int p = class_offset(at, kept, c, &total) + j;
  const unsigned long long key = w.csorted[static_cast<size_t>(c) * at.pre + w.keep[static_cast<size_t>(c) * at.pre + j]];
  // score bits of the class key, then the concatenated position; the class and kept row are found again from p
  w.flat[p] = (key & 0xffffffff00000000ull) | static_cast<unsigned>(p);
}

__global__ void __launch_bounds__(256) a3d_emit_kernel(A3dAttrs at, A3dWs w, float *__restrict__ boxes,
                                                       float *__restrict__ scores, long long *__restrict__ labels,
                                                       int32_t *__restrict__ count) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int32_t *kept = w.cnt + 2 + at.C;
  int total;
  class_offset(at, kept, 0, &total);
  if (p == 0) *count = min(total, at.max_num);
  if (p >= total) return;
  const unsigned long long mine = w.flat[p];
  int rank = p;
  if (total > at.max_num) {
    rank = 0;
    for (int k = 0; k < total; ++k) rank += w.flat[k] < mine;
    if (rank >= at.max_num) return;
  }
  int c = 0, off = 0;
  while (p >= off + kept[c]) off += kept[c++];
  const int j = p - off;
  const unsigned long long key = w.csorted[static_cast<size_t>(c) * at.pre + w.keep[static_cast<size_t>(c) * at.pre + j]];
  const int r = static_cast<int>(key & 0xffffffffull);
  const float *b = w.boxes + static_cast<size_t>(r) * kCode;
  float *ob = boxes + static_cast<size_t>(rank) * kCode;
#pragma unroll
  for (int k = 0; k < kCode; ++k) ob[k] = b[k];
  // limit_period(r - dir_offset, dir_limit_offset, pi) + dir_offset + pi * dir
  const float v = __fsub_rn(b[6], at.dir_off);
  const float fl = floorf(__fadd_rn(__fdiv_rn(v, kPi), at.dir_lim));
  const float lim = __fsub_rn(v, __fmul_rn(fl, kPi));
  ob[6] = __fadd_rn(__fadd_rn(lim, at.dir_off), __fmul_rn(kPi, static_cast<float>(w.dir[r])));
  scores[rank] = __uint_as_float(~static_cast<unsigned>(key >> 32));
  labels[rank] = c;
}

bool sizes(int feat_h, int feat_w, int R, int C, int pre, int max_num, long long *A) {
  if (feat_h < 1 || feat_w < 1 || R < 1 || C < 1 || pre < 1 || max_num < 1) return false;
  *A = static_cast<long long>(feat_h) * feat_w * R;
  return true;
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" size_t p3d_anchor3d_postprocess_workspace_bytes(int feat_h, int feat_w, int anchors_per_loc, int num_classes,
                                                            int nms_pre, int max_num) {
  long long A = 0;
  if (!sizes(feat_h, feat_w, anchors_per_loc, num_classes, nms_pre, max_num, &A)) return 0;
  if (A > 0x7fffffffll || num_classes > kMaxClasses || nms_pre > kMaxPre) return 0;
  return carve(nullptr, A, num_classes, nms_pre, max_num).bytes;
}

extern "C" int p3d_anchor3d_postprocess(const float *head, int feat_h, int feat_w, int anchors_per_loc, int num_classes,
                                        const float *anchors, int nms_pre, float score_thr, float nms_thr, int max_num,
                                        float dir_offset, float dir_limit_offset, float *boxes, float *scores,
                                        int64_t *labels, int32_t *count, void *workspace, size_t workspace_bytes,
                                        p3d_stream_t stream) {
  long long A = 0;
  if (!head || !anchors || !boxes || !scores || !labels || !count ||
      !sizes(feat_h, feat_w, anchors_per_loc, num_classes, nms_pre, max_num, &A) || !(score_thr >= 0.f) ||
      !(nms_thr >= 0.f))
    return P3D_ERR_INVALID_ARG;
  if (A > 0x7fffffffll || num_classes > kMaxClasses || nms_pre > kMaxPre) return P3D_ERR_UNSUPPORTED;
  A3dWs w = carve(workspace, A, num_classes, nms_pre, max_num);
  if (!workspace || workspace_bytes < w.bytes) return P3D_ERR_WORKSPACE;
  A3dAttrs at;
  at.A = static_cast<int>(A);
  at.HW = feat_h * feat_w;
  at.R = anchors_per_loc;
  at.C = num_classes;
  at.pre = nms_pre;
  at.max_num = max_num;
  at.cbmax = (nms_pre + 63) / 64;
  at.cap = nms_pre < max_num ? nms_pre : max_num;
  at.low_bits = 1;
  while (at.low_bits < 32 && ((A - 1) >> at.low_bits)) ++at.low_bits;
  at.score_thr = score_thr;
  at.nms_thr = nms_thr;
  at.dir_off = dir_offset;
  at.dir_lim = dir_limit_offset;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  P3D_CUDA_CHECK(cudaMemsetAsync(w.cnt, 0, sizeof(int32_t) * (2 + 2 * kMaxClasses), st));
  a3d_score_kernel<<<div_up(A, 256), 256, 0, st>>>(head, at, w);
  P3D_LAUNCH_CHECK();
  a3d_select_kernel<<<1, 1024, 0, st>>>(at, w);
  P3D_LAUNCH_CHECK();
  a3d_decode_kernel<<<div_up(nms_pre, 128), 128, 0, st>>>(head, anchors, at, w);
  P3D_LAUNCH_CHECK();
  a3d_sort_kernel<<<num_classes, 1024, 0, st>>>(at, w);
  P3D_LAUNCH_CHECK();
  a3d_mask_kernel<<<dim3(at.cbmax, at.cbmax, num_classes), 64, 0, st>>>(at, w);
  P3D_LAUNCH_CHECK();
  a3d_greedy_kernel<<<num_classes, 256, static_cast<size_t>(at.cbmax) * 8, st>>>(at, w);
  P3D_LAUNCH_CHECK();
  a3d_concat_kernel<<<div_up(static_cast<long long>(num_classes) * at.cap, 256), 256, 0, st>>>(at, w);
  P3D_LAUNCH_CHECK();
  a3d_emit_kernel<<<div_up(static_cast<long long>(num_classes) * at.cap, 256), 256, 0, st>>>(at, w, boxes, scores,
                                                                                         reinterpret_cast<long long *>(labels), count);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
