// Bilinear upsampling of pixel H16 rows (align_corners=True, integer scale), FPN_LSS's nn.Upsample: the x4 of the third
// CustomResNet stage into the 800-channel concat and the x2 before the last two convs (reference: Paddle's
// bilinear_interp_v2 GPU kernel, KeBilinearInterpFw with align_corners).
//
// One thread per (output pixel, 8 channels): the 16 bytes of hi and the 16 bytes of lo' of those channels in each of the
// four source pixels are merged to fp32, interpolated in Paddle's expression with every product and sum rounded on its
// own (__fmul_rn / __fadd_rn: no FMA contraction, so a numpy fp32 restatement matches bit for bit) and split again.
// Scale 1 copies the pairs (FPN_LSS places x0 into the concat with it).  HBM-bound: 4 C h w + 4 C H W bytes.
// Nearest upsampling (CustomFPN's top-down step) copies the pairs of the source pixel, with the same output contract.
#include <cuda_fp16.h>

#include "common.cuh"
#include "h16.cuh"

namespace p3d {
namespace {

struct UpParams {
  const uint8_t *in;
  uint8_t *out;
  int B, h, w, C, H, W, out_C, out_c0, s;
  float ry, rx;  // (in - 1) / (out - 1), 0 for an output extent of 1
  int32_t *status;
};

__global__ void __launch_bounds__(256) upsample_bilinear_h16_kernel(const UpParams p) {
  const int qn = p.C / 8;
  const long long total = static_cast<long long>(p.B) * p.H * p.W * qn;
  const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int q = static_cast<int>(t % qn);
  long long r = t / qn;
  const int X = static_cast<int>(r % p.W);
  r /= p.W;
  const int Y = static_cast<int>(r % p.H);
  const int b = static_cast<int>(r / p.H);
  const size_t in_row = 4 * static_cast<size_t>(p.C), out_row = 4 * static_cast<size_t>(p.out_C);
  const int oc = p.out_c0 + 8 * q;  // first output channel: 16 halfs of hi at (oc / 32) * 128 + (oc % 32) * 2
  uint8_t *o = p.out + ((static_cast<size_t>(b) * p.H + Y) * p.W + X) * out_row + (oc >> 5) * 128 + (oc & 31) * 2;
  const uint8_t *img = p.in + static_cast<size_t>(b) * p.h * p.w * in_row;
  if (p.s == 1) {
    const uint8_t *g = img + (static_cast<size_t>(Y) * p.w + X) * in_row + (q >> 2) * 128 + (q & 3) * 16;
    *reinterpret_cast<uint4 *>(o) = __ldg(reinterpret_cast<const uint4 *>(g));
    *reinterpret_cast<uint4 *>(o + 64) = __ldg(reinterpret_cast<const uint4 *>(g + 64));
    return;
  }
  // bilinear_interp_v2, align_corners: src = ratio * dst, i1 = int(src), i2 = i1 + (i1 < in - 1), l1 = src - i1, l2 = 1 - l1
  const float sy = __fmul_rn(p.ry, static_cast<float>(Y)), sx = __fmul_rn(p.rx, static_cast<float>(X));
  const int y1 = static_cast<int>(sy), x1 = static_cast<int>(sx);
  const int y2 = y1 + (y1 < p.h - 1 ? 1 : 0), x2 = x1 + (x1 < p.w - 1 ? 1 : 0);
  const float h1l = __fsub_rn(sy, static_cast<float>(y1)), h2l = __fsub_rn(1.0f, h1l);
  const float w1l = __fsub_rn(sx, static_cast<float>(x1)), w2l = __fsub_rn(1.0f, w1l);
  float a[8], bb[8], c[8], d[8];
  load8(img + (static_cast<size_t>(y1) * p.w + x1) * in_row, q, a);
  load8(img + (static_cast<size_t>(y1) * p.w + x2) * in_row, q, bb);
  load8(img + (static_cast<size_t>(y2) * p.w + x1) * in_row, q, c);
  load8(img + (static_cast<size_t>(y2) * p.w + x2) * in_row, q, d);
  float v[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float top = __fadd_rn(__fmul_rn(w2l, a[k]), __fmul_rn(w1l, bb[k]));
    const float bot = __fadd_rn(__fmul_rn(w2l, c[k]), __fmul_rn(w1l, d[k]));
    v[k] = __fadd_rn(__fmul_rn(h2l, top), __fmul_rn(h1l, bot));
  }
  bool ovf = false;
  uint4 hi, lo;
  __half2 *h2 = reinterpret_cast<__half2 *>(&hi), *l2 = reinterpret_cast<__half2 *>(&lo);
#pragma unroll
  for (int k = 0; k < 4; ++k) split_h16x2(v[2 * k], v[2 * k + 1], h2[k], l2[k], ovf);
  *reinterpret_cast<uint4 *>(o) = hi;
  *reinterpret_cast<uint4 *>(o + 64) = lo;
  if (ovf && p.status) atomicOr(p.status, 1);
}

// Nearest upsampling by an integer factor (F.interpolate(mode='nearest') to s x the size: source index = dst / s), the
// top-down step of CustomFPN: one thread per (output pixel, 8 channels) copies the 16 bytes of hi and of lo' (exact).
__global__ void __launch_bounds__(256) upsample_nearest_h16_kernel(const UpParams p) {
  const int qn = p.C / 8;
  const long long total = static_cast<long long>(p.B) * p.H * p.W * qn;
  const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int q = static_cast<int>(t % qn);
  long long r = t / qn;
  const int X = static_cast<int>(r % p.W);
  r /= p.W;
  const int Y = static_cast<int>(r % p.H);
  const int b = static_cast<int>(r / p.H);
  const size_t in_row = 4 * static_cast<size_t>(p.C), out_row = 4 * static_cast<size_t>(p.out_C);
  const int oc = p.out_c0 + 8 * q;
  uint8_t *o = p.out + ((static_cast<size_t>(b) * p.H + Y) * p.W + X) * out_row + (oc >> 5) * 128 + (oc & 31) * 2;
  const uint8_t *g = p.in + ((static_cast<size_t>(b) * p.h + Y / p.s) * p.w + X / p.s) * in_row + (q >> 2) * 128 + (q & 3) * 16;
  *reinterpret_cast<uint4 *>(o) = __ldg(reinterpret_cast<const uint4 *>(g));
  *reinterpret_cast<uint4 *>(o + 64) = __ldg(reinterpret_cast<const uint4 *>(g + 64));
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_upsample_bilinear_h16(const void *in_h16, int B, int h, int w, int C, int scale, void *out_h16, int out_C,
                                         int out_c0, int32_t *status_dev, p3d_stream_t stream) {
  if (!in_h16 || !out_h16 || B < 1 || h < 1 || w < 1 || scale < 1 || C < 32 || C % 32 || out_c0 < 0 || out_c0 % 16 ||
      out_C % 32 || out_c0 + C > out_C || (reinterpret_cast<uintptr_t>(in_h16) & 15) || (reinterpret_cast<uintptr_t>(out_h16) & 15))
    return P3D_ERR_INVALID_ARG;
  UpParams p;
  p.in = static_cast<const uint8_t *>(in_h16);
  p.out = static_cast<uint8_t *>(out_h16);
  p.B = B;
  p.h = h;
  p.w = w;
  p.C = C;
  p.H = h * scale;
  p.W = w * scale;
  p.out_C = out_C;
  p.out_c0 = out_c0;
  p.s = scale;
  // Paddle's host ratio: float(in - 1) / (out - 1) with align_corners, 0 for an output of one pixel
  p.ry = p.H > 1 ? static_cast<float>(h - 1) / static_cast<float>(p.H - 1) : 0.f;
  p.rx = p.W > 1 ? static_cast<float>(w - 1) / static_cast<float>(p.W - 1) : 0.f;
  p.status = status_dev;
  const long long total = static_cast<long long>(B) * p.H * p.W * (C / 8);
  upsample_bilinear_h16_kernel<<<div_up(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" int p3d_upsample_nearest_h16(const void *in_h16, int B, int h, int w, int C, int scale, void *out_h16, int out_C,
                                        int out_c0, p3d_stream_t stream) {
  if (!in_h16 || !out_h16 || B < 1 || h < 1 || w < 1 || scale < 1 || C < 32 || C % 32 || out_c0 < 0 || out_c0 % 16 ||
      out_C % 32 || out_c0 + C > out_C || (reinterpret_cast<uintptr_t>(in_h16) & 15) || (reinterpret_cast<uintptr_t>(out_h16) & 15))
    return P3D_ERR_INVALID_ARG;
  UpParams p = {};
  p.in = static_cast<const uint8_t *>(in_h16);
  p.out = static_cast<uint8_t *>(out_h16);
  p.B = B;
  p.h = h;
  p.w = w;
  p.C = C;
  p.H = h * scale;
  p.W = w * scale;
  p.out_C = out_C;
  p.out_c0 = out_c0;
  p.s = scale;
  const long long total = static_cast<long long>(B) * p.H * p.W * (C / 8);
  upsample_nearest_h16_kernel<<<div_up(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
