// BEVDet's test-time image pipeline for sm_90a: Pillow's BICUBIC resize of 8-bit RGB frames, Pillow's crop and
// mmcv.imnormalize, from decoded uint8 HWC frames to the fp32 NCHW images the image encoder reads, in one launch.  The
// result is bit-identical to the host pipeline (PIL.Image.resize + crop, then imnormalize through OpenCV):
//
//   resize     Pillow's ImagingResample on 8 bits per channel: fixed-point coefficients (22 fraction bits, built on the
//              host by ops/image_prep.resize_coeffs), a horizontal pass accumulated in int32 from 1 << 21, >> 22 and
//              clamped into a uint8 intermediate (that rounding is part of Pillow's result), then the vertical pass the
//              same way.  The horizontal pass runs only on the source rows the vertical taps of the kept rows read.
//   crop       rows / columns of the resized image; pixels outside it are 0 (before the normalisation).
//   normalise  fp32(fp64(v -_fp32 mean[c]) * stdinv[c]): cv2.subtract rounds to fp32 with the mean in fp32,
//              cv2.multiply forms the product in fp64 and rounds once.  swap_rb: output channel c is input channel 2 - c
//              (imnormalize's BGR2RGB on an RGB array).
//
// A CTA owns kTH x kTW output pixels of one camera.  It runs the horizontal pass for the tile's kTW resized columns on
// every source row its kTH rows' vertical taps read (the rows' span, at most (kTH - 1) * scale + 2 + taps) into a
// shared uint8 tile (one 32-bit word per pixel: r, g, b, 0), reading the source bytes through the read-only cache, then
// the vertical pass, the clamp and the normalisation, four columns per thread, stored as planar fp32 with 16-byte
// stores when the rows allow it.  Bound by HBM: the band is read about once (tiles share taps through L2) and the
// output is written once.
#include "common.cuh"

namespace p3d {
namespace prep {

constexpr int kTH = 16, kTW = 64;  // output tile
constexpr int kThreads = 256;
constexpr int kPrecision = 22;
static_assert(kTH * kTW / 4 == kThreads, "one thread per four output columns of a tile row");

struct Params {
  const uint8_t *frames;  // [N][band_rows][W0][3]
  const int32_t *kh, *xb, *kv, *yb;
  int N, band_rows, W0, kh_size, rW, kv_size, rH, crop_x, crop_y, fH, fW, span_cap, swap_rb;
  float mean[3];
  double stdinv[3];
  float *out;  // [N][3][fH][fW]
};

__device__ __forceinline__ int clip8(int acc) {
  const int v = acc >> kPrecision;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

__global__ void __launch_bounds__(kThreads) image_prep_u8_kernel(const Params p) {
  extern __shared__ __align__(16) uint8_t smem[];
  int32_t *kh_s = reinterpret_cast<int32_t *>(smem);  // [kTW][kh_size]
  int32_t *kv_s = kh_s + kTW * p.kh_size;              // [kTH][kv_size]
  int2 *xb_s = reinterpret_cast<int2 *>(kv_s + kTH * p.kv_size);
  int2 *yb_s = xb_s + kTW;
  uint32_t *hs = reinterpret_cast<uint32_t *>(yb_s + kTH);  // [span_cap][kTW]
  const int tid = threadIdx.x, b = blockIdx.z;
  const int ox0 = blockIdx.x * kTW, oy0 = blockIdx.y * kTH;

  for (int i = tid; i < kTW; i += kThreads) {
    const int rx = p.crop_x + ox0 + i;
    const bool in = ox0 + i < p.fW && rx >= 0 && rx < p.rW;
    xb_s[i] = in ? make_int2(__ldg(p.xb + 2 * rx), __ldg(p.xb + 2 * rx + 1)) : make_int2(0, 0);
  }
  for (int i = tid; i < kTW * p.kh_size; i += kThreads) {
    const int c = i / p.kh_size, rx = p.crop_x + ox0 + c;
    kh_s[i] = (ox0 + c < p.fW && rx >= 0 && rx < p.rW) ? __ldg(p.kh + static_cast<size_t>(rx) * p.kh_size + i % p.kh_size) : 0;
  }
  for (int i = tid; i < kTH; i += kThreads) {
    const int ry = p.crop_y + oy0 + i;
    const bool in = oy0 + i < p.fH && ry >= 0 && ry < p.rH;
    yb_s[i] = in ? make_int2(__ldg(p.yb + 2 * ry), __ldg(p.yb + 2 * ry + 1)) : make_int2(0, 0);
  }
  for (int i = tid; i < kTH * p.kv_size; i += kThreads) {
    const int r = i / p.kv_size, ry = p.crop_y + oy0 + r;
    kv_s[i] = (oy0 + r < p.fH && ry >= 0 && ry < p.rH) ? __ldg(p.kv + static_cast<size_t>(ry) * p.kv_size + i % p.kv_size) : 0;
  }
  // the tile's kept rows are contiguous: local rows [r_first, r_last]
  const int r_first = max(0, -p.crop_y - oy0);
  const int r_last = min(min(kTH, p.fH - oy0), p.rH - p.crop_y - oy0) - 1;
  __syncthreads();

  int sy0 = 0, span = 0;
  if (r_first <= r_last) {
    sy0 = yb_s[r_first].x;
    span = min(yb_s[r_last].x + yb_s[r_last].y - sy0, p.span_cap);
  }
  // horizontal pass: (source row sy0 + r, tile column c) -> uint8 r, g, b
  const uint8_t *img = p.frames + static_cast<size_t>(b) * p.band_rows * p.W0 * 3;
  for (int i = tid; i < span * kTW; i += kThreads) {
    const int r = i / kTW, c = i % kTW;
    const int sy = sy0 + r;
    const int2 xb = xb_s[c];
    uint32_t word = 0u;
    if (xb.y > 0 && sy >= 0 && sy < p.band_rows) {
      const uint8_t *src = img + (static_cast<size_t>(sy) * p.W0 + xb.x) * 3;
      const int32_t *k = kh_s + c * p.kh_size;
      int a0 = 1 << (kPrecision - 1), a1 = a0, a2 = a0;
      for (int t = 0; t < xb.y; ++t) {
        const int w = k[t];
        a0 += static_cast<int>(__ldg(src + 3 * t)) * w;
        a1 += static_cast<int>(__ldg(src + 3 * t + 1)) * w;
        a2 += static_cast<int>(__ldg(src + 3 * t + 2)) * w;
      }
      word = static_cast<uint32_t>(clip8(a0)) | (static_cast<uint32_t>(clip8(a1)) << 8) |
             (static_cast<uint32_t>(clip8(a2)) << 16);
    }
    hs[r * kTW + c] = word;
  }
  __syncthreads();

  // vertical pass, clamp, normalise: local row lr, columns 4 q .. 4 q + 3
  const int lr = tid / (kTW / 4), q = tid % (kTW / 4);
  const int oy = oy0 + lr;
  if (oy >= p.fH) return;
  const bool row_in = lr >= r_first && lr <= r_last;
  const int2 yb = yb_s[lr];
  const int32_t *k = kv_s + lr * p.kv_size;
  int v[4][3];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = 4 * q + j;
    v[j][0] = v[j][1] = v[j][2] = 0;
    if (!row_in || xb_s[c].y == 0) continue;  // outside the resized image (or past fW): Pillow's crop fills 0
    int a0 = 1 << (kPrecision - 1), a1 = a0, a2 = a0;
    for (int t = 0; t < yb.y; ++t) {
      const int r = yb.x - sy0 + t;
      const uint32_t w8 = (r >= 0 && r < span) ? hs[r * kTW + c] : 0u;
      const int w = k[t];
      a0 += static_cast<int>(w8 & 0xffu) * w;
      a1 += static_cast<int>((w8 >> 8) & 0xffu) * w;
      a2 += static_cast<int>((w8 >> 16) & 0xffu) * w;
    }
    v[j][0] = clip8(a0);
    v[j][1] = clip8(a1);
    v[j][2] = clip8(a2);
  }
  const int ox = ox0 + 4 * q;
  if (ox >= p.fW) return;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const int ic = p.swap_rb ? 2 - ch : ch;
    float f[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int x = ic == 0 ? v[j][0] : (ic == 1 ? v[j][1] : v[j][2]);
      f[j] = __double2float_rn(static_cast<double>(__fsub_rn(static_cast<float>(x), p.mean[ch])) * p.stdinv[ch]);
    }
    float *o = p.out + ((static_cast<size_t>(b) * 3 + ch) * p.fH + oy) * p.fW + ox;
    if ((p.fW & 3) == 0) {  // fW % 4 == 0: ox % 4 == 0 and the whole quad is inside the row
      *reinterpret_cast<float4 *>(o) = make_float4(f[0], f[1], f[2], f[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (ox + j < p.fW) o[j] = f[j];
    }
  }
}

// Pillow's tap count for a resize from in_size to out_size pixels: 2 * ceil(2 * max(in / out, 1)) + 1
inline int taps(int in_size, int out_size) {
  double fs = static_cast<double>(in_size) / out_size;
  if (fs < 1.0) fs = 1.0;
  return static_cast<int>(ceil(2.0 * fs)) * 2 + 1;
}

}  // namespace prep
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_image_prep_u8(const uint8_t *frames, int N, int band_rows, int H0, int W0, const int32_t *kh,
                                 const int32_t *xbounds, int kh_size, int rW, const int32_t *kv, const int32_t *ybounds,
                                 int kv_size, int rH, int crop_x, int crop_y, int fH, int fW, const float *mean_host,
                                 const double *std_inv_host, int swap_rb, float *out, p3d_stream_t stream) {
  if (!frames || !kh || !xbounds || !kv || !ybounds || !mean_host || !std_inv_host || !out) return P3D_ERR_INVALID_ARG;
  if (N < 1 || band_rows < 1 || H0 < 1 || W0 < 1 || rW < 1 || rH < 1 || fH < 1 || fW < 1 || kh_size < 1 || kv_size < 1 ||
      band_rows > H0 || (reinterpret_cast<uintptr_t>(out) & 15))
    return P3D_ERR_INVALID_ARG;
  if (crop_x < -(1 << 28) || crop_x > (1 << 28) || crop_y < -(1 << 28) || crop_y > (1 << 28)) return P3D_ERR_INVALID_ARG;
  if (W0 > 8ll * rW || H0 > 8ll * rH) return P3D_ERR_UNSUPPORTED;  // more than 33 taps
  if (kh_size != prep::taps(W0, rW) || kv_size != prep::taps(H0, rH)) return P3D_ERR_INVALID_ARG;
  if (static_cast<long long>(N) * 3 * fH * fW >= (1ll << 31) || N > 65535) return P3D_ERR_UNSUPPORTED;
  prep::Params p;
  p.frames = frames;
  p.kh = kh;
  p.xb = xbounds;
  p.kv = kv;
  p.yb = ybounds;
  p.N = N;
  p.band_rows = band_rows;
  p.W0 = W0;
  p.kh_size = kh_size;
  p.rW = rW;
  p.kv_size = kv_size;
  p.rH = rH;
  p.crop_x = crop_x;
  p.crop_y = crop_y;
  p.fH = fH;
  p.fW = fW;
  // source rows under kTH consecutive output rows: their first taps advance by at most ceil((kTH - 1) * scale) + 1
  p.span_cap = static_cast<int>(ceil((prep::kTH - 1) * static_cast<double>(H0) / rH)) + 1 + kv_size;
  p.swap_rb = swap_rb ? 1 : 0;
  for (int c = 0; c < 3; ++c) {
    p.mean[c] = mean_host[c];
    p.stdinv[c] = std_inv_host[c];
  }
  p.out = out;
  const size_t smem = static_cast<size_t>(prep::kTW * kh_size + prep::kTH * kv_size) * 4 +
                      static_cast<size_t>(prep::kTW + prep::kTH) * 8 + static_cast<size_t>(p.span_cap) * prep::kTW * 4;
  const dim3 grid(div_up(fW, prep::kTW), div_up(fH, prep::kTH), N);
  if (grid.y > 65535) return P3D_ERR_UNSUPPORTED;
  if (smem > 48 * 1024)
    P3D_CUDA_CHECK(cudaFuncSetAttribute(prep::image_prep_u8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(smem)));
  prep::image_prep_u8_kernel<<<grid, prep::kThreads, smem, static_cast<cudaStream_t>(stream)>>>(p);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
