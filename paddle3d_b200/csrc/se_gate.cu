// BEVFusion's SE_Block (x * sigmoid(Conv1x1_bias(mean_hw(x)))) on a pixel H16 image, in place, as four launches:
//   S1 se_partial  each CTA sums the channels of kPixPerCta consecutive pixels in fp64 and writes one partial row
//   S2 se_mean     per channel, the partial rows summed in index order, divided by H * W (no atomics anywhere, so the
//                  mean and everything after it are bit-reproducible)
//   S3 se_fc       one warp per output channel: bias + weight[o, :] . mean in fp64 (lanes over c, the lane sums
//                  combined in a fixed shuffle order), sigmoid in fp64, rounded to the fp32 gate
//   S4 se_scale    x = fp32(hi + lo'), x * gate in fp32, split again (the reference multiplies an fp32 tensor by an fp32
//                  gate: one rounding); status bit 0 when a value leaves fp16's range.
// The gate conv is a C x C matrix-vector product per image, not an image conv, so it is not run through the dense conv.
#include "common.cuh"
#include "h16.cuh"

namespace p3d {
namespace {

constexpr int kPixPerCta = 128;
constexpr int kMaxC = 1024;
constexpr int kRows = 4;  // pixel lanes of an S1 CTA: kRows x kMaxC doubles of shared memory

int chunks(long long HW) { return static_cast<int>(div_up(HW, kPixPerCta)); }

struct SeWs {
  double *partial;  // [B, chunks, C]
  double *mean;     // [B, C]
  size_t bytes;
};

SeWs carve(void *p, int B, long long HW, int C) {
  SeWs w;
  Carver c(p);
  w.partial = c.take<double>(static_cast<size_t>(B) * chunks(HW) * C);
  w.mean = c.take<double>(static_cast<size_t>(B) * C);
  w.bytes = c.off;
  return w;
}

// block (32, kRows): x over 8-channel groups q, y over pixels; grid (chunks, B)
__global__ void __launch_bounds__(256) se_partial_kernel(const uint8_t *__restrict__ img, long long HW, int C,
                                                         double *__restrict__ partial) {
  __shared__ double s_sum[kRows][kMaxC];
  const int b = blockIdx.y, Q = C / 8;
  const long long p0 = static_cast<long long>(blockIdx.x) * kPixPerCta;
  const long long p1 = min(p0 + kPixPerCta, HW);
  const size_t row_bytes = static_cast<size_t>(C) * 4;
  for (int q = threadIdx.x; q < Q; q += 32) {
    double acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll 4
    for (long long p = p0 + threadIdx.y; p < p1; p += kRows) {
      float v[8];
      load8(img + (static_cast<size_t>(b) * HW + p) * row_bytes, q, v);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += static_cast<double>(v[k]);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) s_sum[threadIdx.y][q * 8 + k] = acc[k];
  }
  __syncthreads();
  double *out = partial + (static_cast<size_t>(b) * gridDim.x + blockIdx.x) * C;
  for (int c = threadIdx.y * 32 + threadIdx.x; c < C; c += 32 * kRows) {
    double s = 0.0;
#pragma unroll
    for (int r = 0; r < kRows; ++r) s += s_sum[r][c];
    out[c] = s;
  }
}

__global__ void __launch_bounds__(256) se_mean_kernel(const double *__restrict__ partial, int nchunk, long long HW, int C,
                                                      double *__restrict__ mean) {
  const int b = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double *p = partial + static_cast<size_t>(b) * nchunk * C + c;
  double s = 0.0;
#pragma unroll 8
  for (int k = 0; k < nchunk; ++k) s += p[static_cast<size_t>(k) * C];
  mean[static_cast<size_t>(b) * C + c] = s / static_cast<double>(HW);
}

// 8 warps per CTA, one output channel per warp; grid (div_up(C, 8), B)
__global__ void __launch_bounds__(256) se_fc_kernel(const double *__restrict__ mean, int C, const float *__restrict__ weight,
                                                    const float *__restrict__ bias, float *__restrict__ gate) {
  const int b = blockIdx.y, lane = threadIdx.x & 31, o = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (o >= C) return;
  const double *m = mean + static_cast<size_t>(b) * C;
  const float *wr = weight + static_cast<size_t>(o) * C;
  double acc = 0.0;
  for (int c = lane; c < C; c += 32) acc = fma(static_cast<double>(__ldg(wr + c)), m[c], acc);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
  if (lane == 0) gate[static_cast<size_t>(b) * C + o] = static_cast<float>(1.0 / (1.0 + exp(-(acc + bias[o]))));
}

// one thread per (pixel, 8-channel group q); grid (div_up(HW * Q, 256), B)
__global__ void __launch_bounds__(256) se_scale_kernel(uint8_t *__restrict__ img, long long HW, int C,
                                                       const float *__restrict__ gate, int32_t *__restrict__ status) {
  const int b = blockIdx.y, Q = C / 8;
  const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  bool ovf = false;
  if (e < HW * Q) {
    const long long p = e / Q;
    const int q = static_cast<int>(e - p * Q);
    uint8_t *g = img + (static_cast<size_t>(b) * HW + p) * C * 4 + (q >> 2) * 128 + (q & 3) * 16;
    uint4 hi = *reinterpret_cast<const uint4 *>(g), lo = *reinterpret_cast<const uint4 *>(g + 64);
    __half2 *h2 = reinterpret_cast<__half2 *>(&hi), *l2 = reinterpret_cast<__half2 *>(&lo);
    const float *gt = gate + static_cast<size_t>(b) * C + q * 8;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 fh = __half22float2(h2[k]), fl = __half22float2(l2[k]);
      const float a = __fmul_rn(fmaf(fl.x, kLoInv, fh.x), __ldg(gt + 2 * k));
      const float c = __fmul_rn(fmaf(fl.y, kLoInv, fh.y), __ldg(gt + 2 * k + 1));
      split_h16x2(a, c, h2[k], l2[k], ovf);
    }
    *reinterpret_cast<uint4 *>(g) = hi;
    *reinterpret_cast<uint4 *>(g + 64) = lo;
  }
  if (__any_sync(0xffffffffu, ovf) && (threadIdx.x & 31) == 0) atomicOr(status, 1);
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" size_t p3d_se_gate_workspace_bytes(int B, int H, int W, int C) {
  if (B < 1 || H < 1 || W < 1 || C < 1) return 0;
  return carve(nullptr, B, static_cast<long long>(H) * W, C).bytes;
}

extern "C" int p3d_se_gate_h16(void *img_h16, int B, int H, int W, int C, const float *weight, const float *bias,
                               float *gate_dev, int32_t *status_dev, void *workspace, size_t workspace_bytes,
                               p3d_stream_t stream) {
  if (!img_h16 || !weight || !bias || !gate_dev || !status_dev || B < 1 || H < 1 || W < 1 || C < 32 || C % 32 ||
      (reinterpret_cast<uintptr_t>(img_h16) & 15))
    return P3D_ERR_INVALID_ARG;
  if (C > kMaxC || B > 65535) return P3D_ERR_UNSUPPORTED;
  const long long HW = static_cast<long long>(H) * W;
  if (HW * (C / 8) >= (1ll << 31) * 256) return P3D_ERR_UNSUPPORTED;
  SeWs w = carve(workspace, B, HW, C);
  if (!workspace || workspace_bytes < w.bytes) return P3D_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t *img = static_cast<uint8_t *>(img_h16);
  const int nchunk = chunks(HW);
  se_partial_kernel<<<dim3(nchunk, B), dim3(32, kRows), 0, st>>>(img, HW, C, w.partial);
  P3D_LAUNCH_CHECK();
  se_mean_kernel<<<dim3(div_up(C, 256), B), 256, 0, st>>>(w.partial, nchunk, HW, C, w.mean);
  P3D_LAUNCH_CHECK();
  se_fc_kernel<<<dim3(div_up(C, 8), B), 256, 0, st>>>(w.mean, C, weight, bias, gate_dev);
  P3D_LAUNCH_CHECK();
  se_scale_kernel<<<dim3(div_up(HW * (C / 8), 256), B), 256, 0, st>>>(img, HW, C, gate_dev, status_dev);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
