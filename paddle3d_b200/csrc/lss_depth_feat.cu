// Depth softmax + feature permute of LSSViewTransformer (bevdet_transformer.py:305-316 softmax, :192-228 permute), one
// launch.  A block owns 32 consecutive pixels of one camera: it stages their D logits in shared memory (coalesced over
// the pixels), 32 threads take the max and the sum over d in ascending order, then all threads write
// expf(x - max) / sum; then the C x 32 tile of tran_feat is staged and written out as the contiguous [32, C] slice of feat.
// Algorithmic bytes: 8 * BN * (D + C) * H * W (each tensor read once and written once).  Bound: latency.  At the BEVDet
// shape there are only BN * H * W = 4224 pixels, each a serial 118-term max / expf / sum chain, in 132 blocks.
#include <cuda_fp16.h>

#include "common.cuh"
#include "h16.cuh"

namespace p3d {
namespace {

constexpr int kPix = 32;
constexpr int kSmemFloats = 12 * 1024 - 2 * kPix;  // 48 KB with the max / sum: D * 32 and C * 33 floats must fit

__global__ void __launch_bounds__(256) lss_depth_feat_kernel(const float *__restrict__ logits, const float *__restrict__ tf,
                                                             int D, int HW, int C, float *__restrict__ depth,
                                                             float *__restrict__ feat) {
  __shared__ float sm[kSmemFloats];
  __shared__ float mx[kPix], sum[kPix];
  const long long bn = blockIdx.y;
  const int p0 = blockIdx.x * kPix;
  const int np = min(kPix, HW - p0);
  const float *lg = logits + bn * D * HW + p0;
  for (int i = threadIdx.x; i < D * kPix; i += blockDim.x) {
    const int d = i / kPix, p = i % kPix;
    sm[i] = p < np ? __ldg(lg + static_cast<size_t>(d) * HW + p) : 0.f;
  }
  __syncthreads();
  if (threadIdx.x < kPix) {
    const int p = threadIdx.x;
    float m = sm[p];
    for (int d = 1; d < D; ++d) m = fmaxf(m, sm[d * kPix + p]);
    float s = 0.f;
    for (int d = 0; d < D; ++d) s = __fadd_rn(s, expf(__fsub_rn(sm[d * kPix + p], m)));
    mx[p] = m;
    sum[p] = s;
  }
  __syncthreads();
  float *dp = depth + bn * D * HW + p0;
  for (int i = threadIdx.x; i < D * kPix; i += blockDim.x) {
    const int d = i / kPix, p = i % kPix;
    if (p < np) dp[static_cast<size_t>(d) * HW + p] = __fdiv_rn(expf(__fsub_rn(sm[i], mx[p])), sum[p]);
  }
  __syncthreads();
  const float *src = tf + bn * C * HW + p0;
  for (int i = threadIdx.x; i < C * kPix; i += blockDim.x) {
    const int c = i / kPix, p = i % kPix;
    sm[c * (kPix + 1) + p] = p < np ? __ldg(src + static_cast<size_t>(c) * HW + p) : 0.f;
  }
  __syncthreads();
  float *fo = feat + (bn * HW + p0) * C;
  for (int i = threadIdx.x; i < np * C; i += blockDim.x) {
    const int p = i / C, c = i % C;
    fo[i] = sm[c * (kPix + 1) + p];
  }
}

// The same step from the depth net's pixel fp16-pair rows [BN * HW][in_C channels] (channels [0, D) the logits, [D, D + C)
// the features, merged as pixel_h16_to_nchw merges them): the block stages its 32 pixels' logits at pitch 33 (threads run
// along a pixel's channels), then the softmax of lss_depth_feat_kernel with the same operations in the same order, then
// feat straight from the rows.
constexpr int kPitch = kPix + 1;

__device__ __forceinline__ float pair_at(const __half *row, int c) { return merge_h16(row[(c >> 5) * 64 + (c & 31)], row[(c >> 5) * 64 + 32 + (c & 31)]); }

__global__ void __launch_bounds__(256) lss_depth_feat_h16_kernel(const __half *__restrict__ rows, int in_C, int D, int HW, int C,
                                                                 float *__restrict__ depth, float *__restrict__ feat) {
  __shared__ float sm[kSmemFloats];
  __shared__ float mx[kPix], sum[kPix];
  const long long bn = blockIdx.y;
  const int p0 = blockIdx.x * kPix;
  const int np = min(kPix, HW - p0);
  const __half *px = rows + (bn * HW + p0) * 2 * in_C;
  for (int i = threadIdx.x; i < D * kPix; i += blockDim.x) {
    const int p = i / D, d = i % D;
    sm[d * kPitch + p] = p < np ? pair_at(px + static_cast<size_t>(p) * 2 * in_C, d) : 0.f;
  }
  __syncthreads();
  if (threadIdx.x < kPix) {
    const int p = threadIdx.x;
    float m = sm[p];
    for (int d = 1; d < D; ++d) m = fmaxf(m, sm[d * kPitch + p]);
    float s = 0.f;
    for (int d = 0; d < D; ++d) s = __fadd_rn(s, expf(__fsub_rn(sm[d * kPitch + p], m)));
    mx[p] = m;
    sum[p] = s;
  }
  __syncthreads();
  float *dp = depth + bn * D * HW + p0;
  for (int i = threadIdx.x; i < D * kPix; i += blockDim.x) {
    const int d = i / kPix, p = i % kPix;
    if (p < np) dp[static_cast<size_t>(d) * HW + p] = __fdiv_rn(expf(__fsub_rn(sm[d * kPitch + p], mx[p])), sum[p]);
  }
  float *fo = feat + (bn * HW + p0) * C;
  for (int i = threadIdx.x; i < np * C; i += blockDim.x) {
    const int p = i / C, c = i % C;
    fo[i] = pair_at(px + static_cast<size_t>(p) * 2 * in_C, D + c);
  }
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_lss_depth_feat_h16(const void *rows_h16, int BN, int H, int W, int in_C, int D, int C, float *depth,
                                      float *feat, p3d_stream_t stream) {
  if (!rows_h16 || !depth || !feat || BN < 1 || D < 1 || H < 1 || W < 1 || C < 1 || in_C < 32 || in_C % 32 || D + C > in_C ||
      (reinterpret_cast<uintptr_t>(rows_h16) & 15))
    return P3D_ERR_INVALID_ARG;
  const long long hw = static_cast<long long>(H) * W;
  constexpr int kMaxD = kSmemFloats / kPitch;  // 370
  if (D > kMaxD || BN > 65535 || static_cast<long long>(BN) * hw * 2 * in_C > 0x7fffffffll ||
      static_cast<long long>(BN) * (D > C ? D : C) * hw > 0x7fffffffll)
    return P3D_ERR_UNSUPPORTED;
  const dim3 grid(div_up(hw, kPix), BN);
  lss_depth_feat_h16_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const __half *>(rows_h16), in_C, D,
                                                                                static_cast<int>(hw), C, depth, feat);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" int p3d_lss_depth_feat(const float *logits, const float *tran_feat, int BN, int D, int H, int W, int C, float *depth,
                                  float *feat, p3d_stream_t stream) {
  if (!logits || !tran_feat || !depth || !feat || BN < 1 || D < 1 || H < 1 || W < 1 || C < 1) return P3D_ERR_INVALID_ARG;
  const long long hw = static_cast<long long>(H) * W;
  constexpr int kMaxD = kSmemFloats / kPix, kMaxC = kSmemFloats / (kPix + 1);  // 382, 370
  if (D > kMaxD || C > kMaxC || BN > 65535 ||
      static_cast<long long>(BN) * (D > C ? D : C) * hw > 0x7fffffffll)
    return P3D_ERR_UNSUPPORTED;
  const dim3 grid(div_up(hw, kPix), BN);
  lss_depth_feat_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(logits, tran_feat, D, static_cast<int>(hw), C,
                                                                            depth, feat);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
