// BEVDet4D's shift_feature on pixel H16 rows: the previous frame's BEV resampled into the current ego frame,
// F.grid_sample(feat_prev, grid, mode='bilinear', padding_mode='zeros', align_corners=True) with the grid of the affine
// BEV-pixel transform tf (gen_grid: grid = tf (x, y, 1), normalised by / (W - 1) * 2 - 1).
//
// One thread per (output pixel, 8 channels), as upsample.cu: the sample coordinate in the reference's fp32 chain with
// every product and sum rounded on its own (__fmul_rn / __fadd_rn / __fdiv_rn: no contraction, so a numpy fp32
// restatement matches bit for bit), grid_sample's unnormalisation, floor, the four weights and the sum
// nw NW + ne NE + sw SW + se SE in that order, then the split.  A tap outside the image contributes 0 and is not read;
// the in-range test runs on the floats, so NaN / huge coordinates never reach an integer conversion.  The transform is
// read on the device, so one captured graph serves every ego motion.  HBM / L2-bound: 4 C h w + 4 C h w bytes.
#include <cuda_fp16.h>

#include "common.cuh"
#include "h16.cuh"

namespace p3d {
namespace {

struct ShiftParams {
  const uint8_t *in;
  uint8_t *out;
  const float *tf;  // [B, 6]
  int B, h, w, in_C, C, out_C, out_c0;
  int32_t *status;
};

__global__ void __launch_bounds__(256) bev_shift_h16_kernel(const ShiftParams p) {
  const int qn = p.C / 8;
  const long long total = static_cast<long long>(p.B) * p.h * p.w * qn;
  const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int q = static_cast<int>(t % qn);
  long long r = t / qn;
  const int X = static_cast<int>(r % p.w);
  r /= p.w;
  const int Y = static_cast<int>(r % p.h);
  const int b = static_cast<int>(r / p.h);
  const float *tf = p.tf + 6 * b;
  const float fx = static_cast<float>(X), fy = static_cast<float>(Y);
  // gen_grid: g = tf (x, y, 1), then / (W - 1) * 2 - 1
  const float gx = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(tf + 0), fx), __fmul_rn(__ldg(tf + 1), fy)), __ldg(tf + 2));
  const float gy = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(tf + 3), fx), __fmul_rn(__ldg(tf + 4), fy)), __ldg(tf + 5));
  const float wm1 = static_cast<float>(p.w - 1), hm1 = static_cast<float>(p.h - 1);
  const float nx = __fsub_rn(__fmul_rn(__fdiv_rn(gx, wm1), 2.0f), 1.0f);
  const float ny = __fsub_rn(__fmul_rn(__fdiv_rn(gy, hm1), 2.0f), 1.0f);
  // grid_sample, align_corners: ((g + 1) / 2) * (size - 1)
  const float ix = __fmul_rn(__fmul_rn(__fadd_rn(nx, 1.0f), 0.5f), wm1);
  const float iy = __fmul_rn(__fmul_rn(__fadd_rn(ny, 1.0f), 0.5f), hm1);
  const float x0 = floorf(ix), y0 = floorf(iy);
  const float x1 = __fadd_rn(x0, 1.0f), y1 = __fadd_rn(y0, 1.0f);
  const float dxl = __fsub_rn(ix, x0), dxr = __fsub_rn(x1, ix), dyt = __fsub_rn(iy, y0), dyb = __fsub_rn(y1, iy);
  const float wnw = __fmul_rn(dxr, dyb), wne = __fmul_rn(dxl, dyb), wsw = __fmul_rn(dxr, dyt), wse = __fmul_rn(dxl, dyt);
  // in-range tests on the floats (false for NaN); indices clamped before the conversion
  const bool vx0 = x0 >= 0.0f && x0 <= wm1, vx1 = x1 >= 0.0f && x1 <= wm1;
  const bool vy0 = y0 >= 0.0f && y0 <= hm1, vy1 = y1 >= 0.0f && y1 <= hm1;
  const int ix0 = static_cast<int>(fminf(fmaxf(x0, 0.0f), wm1)), ix1 = static_cast<int>(fminf(fmaxf(x1, 0.0f), wm1));
  const int iy0 = static_cast<int>(fminf(fmaxf(y0, 0.0f), hm1)), iy1 = static_cast<int>(fminf(fmaxf(y1, 0.0f), hm1));
  const size_t in_row = 4 * static_cast<size_t>(p.in_C), out_row = 4 * static_cast<size_t>(p.out_C);
  const uint8_t *img = p.in + static_cast<size_t>(b) * p.h * p.w * in_row;
  float v[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) v[k] = 0.0f;
  const bool valid[4] = {vx0 && vy0, vx1 && vy0, vx0 && vy1, vx1 && vy1};
  const int tx[4] = {ix0, ix1, ix0, ix1}, ty[4] = {iy0, iy0, iy1, iy1};
  const float wt[4] = {wnw, wne, wsw, wse};
#pragma unroll
  for (int c = 0; c < 4; ++c) {  // nw, ne, sw, se
    float a[8];
    if (valid[c]) {
      load8(img + (static_cast<size_t>(ty[c]) * p.w + tx[c]) * in_row, q, a);
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) a[k] = 0.0f;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = __fadd_rn(v[k], valid[c] ? __fmul_rn(wt[c], a[k]) : 0.0f);
  }
  bool ovf = false;
  uint4 hi, lo;
  __half2 *h2 = reinterpret_cast<__half2 *>(&hi), *l2 = reinterpret_cast<__half2 *>(&lo);
#pragma unroll
  for (int k = 0; k < 4; ++k) split_h16x2(v[2 * k], v[2 * k + 1], h2[k], l2[k], ovf);
  const int oc = p.out_c0 + 8 * q;  // first output channel: 16 halfs of hi at (oc / 32) * 128 + (oc % 32) * 2
  uint8_t *o = p.out + ((static_cast<size_t>(b) * p.h + Y) * p.w + X) * out_row + (oc >> 5) * 128 + (oc & 31) * 2;
  *reinterpret_cast<uint4 *>(o) = hi;
  *reinterpret_cast<uint4 *>(o + 64) = lo;
  if (ovf && p.status) atomicOr(p.status, 1);
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_bev_shift_h16(const void *in_h16, int B, int h, int w, int in_C, int C, const float *tf_dev, void *out_h16,
                                 int out_C, int out_c0, int32_t *status_dev, p3d_stream_t stream) {
  if (!in_h16 || !out_h16 || !tf_dev || B < 1 || h < 2 || w < 2 || C < 16 || C % 16 || C > in_C || in_C % 32 ||
      out_C % 32 || out_c0 < 0 || out_c0 % 16 || out_c0 + C > out_C || (reinterpret_cast<uintptr_t>(in_h16) & 15) ||
      (reinterpret_cast<uintptr_t>(out_h16) & 15) || (reinterpret_cast<uintptr_t>(tf_dev) & 3))
    return P3D_ERR_INVALID_ARG;
  ShiftParams p;
  p.in = static_cast<const uint8_t *>(in_h16);
  p.out = static_cast<uint8_t *>(out_h16);
  p.tf = tf_dev;
  p.B = B;
  p.h = h;
  p.w = w;
  p.in_C = in_C;
  p.C = C;
  p.out_C = out_C;
  p.out_c0 = out_c0;
  p.status = status_dev;
  const long long total = static_cast<long long>(B) * h * w * (C / 8);
  bev_shift_h16_kernel<<<div_up(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
