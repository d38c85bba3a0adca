// ResNet stem of BEVDet's image backbone (mmdet ResNet, style 'pytorch'): conv 7x7 stride 2 pad 3, 3 -> 64, BatchNorm
// (eval, folded into scale / shift), ReLU and MaxPool2d(3, 2, 1), in one launch, from fp32 NCHW images to pixel
// fp16-pair rows [B * pH * pW][64 channels: 2 groups of hi 32 | lo' 32].
//
// A CTA owns an 8 x 16 tile of pooled outputs.  It needs the 17 x 33 conv outputs under their pool windows (the one-pixel
// pool halo included) and the 39 x 71 x 3 input patch under those.  The patch is split once into (hi, lo') fp16 pairs
// (one 32-bit word per element: hi in the low half) in shared memory; the conv is an implicit GEMM [561 conv pixels] x
// [K = 3 * 49 = 147, padded to 160] x [64 channels] on warp mma.sync.m16n8k16, each A fragment gathered from the patch
// through a per-k offset table.  Both operands are fp16 pairs: acc = hi.hi + (hi.lo' + lo'.hi) 2^-11, the three
// products of the other fp16-pair kernels, the two lo' products in one fp32 accumulator.  The epilogue applies
// fma(acc, scale, shift) and ReLU and max-reduces each conv output into the pooled cells whose 3 x 3 windows hold it, with
// a 32-bit atomicMax on the float bits in shared memory (exact: after ReLU every value is >= +0, where the bit order is
// the value order; conv pixels outside the conv image take no part, as MaxPool's -inf padding).  The pooled fp32 tile is
// split once and stored.  The 128 x 352 x 64 conv image never leaves the SM.
//
// Weights: p3d_resnet_stem_pack_weights lays W [64][3][7][7] out in mma B-fragment order, [10 k-steps][8 n-tiles][32
// lanes] x (hi b0, hi b1, lo' b0, lo' b1), 40 KB, which every CTA copies to shared memory once.
#include <cuda_fp16.h>

#include "common.cuh"
#include "h16.cuh"
#include "tc_common.cuh"

namespace p3d {
namespace stem {

constexpr int kCin = 3, kK = 7, kCout = 64;
constexpr int kKReal = kCin * kK * kK;        // 147
constexpr int kSteps = 10;                    // k-steps of 16: K padded to 160
constexpr int kPH = 8, kPW = 16;              // pooled tile
constexpr int kCR = 2 * kPH + 1, kCC = 2 * kPW + 1;  // conv tile 17 x 33
constexpr int kConvPx = kCR * kCC;            // 561
constexpr int kMTiles = (kConvPx + 15) / 16;  // 36
constexpr int kIR = 2 * kCR + 5, kIC = 2 * kCC + 5;  // input patch 39 x 71
constexpr int kIP = 72;                       // patch pitch (words)
constexpr int kPatchWords = kCin * kIR * kIP;
constexpr int kPoolPitch = kCout + 1;         // pooled cell pitch (words): odd, spreads the atomics over the banks
constexpr int kThreads = 256, kWarps = kThreads / 32;
constexpr int kWeightU4 = kSteps * 8 * 32;    // 2560 uint4 = 40 KB
constexpr size_t kSmemBytes = static_cast<size_t>(kWeightU4) * 16 + static_cast<size_t>(kPatchWords) * 4 +
                              static_cast<size_t>(kPH * kPW * kPoolPitch) * 4 + kSteps * 4 * 16;

struct Params {
  const float *in;      // [B][3][H][W]
  const uint4 *packed;  // [kSteps][8][32]
  const float *scale, *shift;
  uint8_t *out;         // [B][pH][pW][256 bytes]
  int B, H, W, cH, cW, pH, pW;
  int32_t *status;
};

__device__ __forceinline__ uint32_t pair_word(float x, bool &ovf) {
  __half hi, lo;
  split_h16(x, hi, lo, ovf);
  return static_cast<uint32_t>(__half_as_ushort(hi)) | (static_cast<uint32_t>(__half_as_ushort(lo)) << 16);
}

__global__ void __launch_bounds__(kThreads, 2) resnet_stem_h16_kernel(const Params p) {
  extern __shared__ __align__(16) uint8_t smem[];
  uint4 *wsm = reinterpret_cast<uint4 *>(smem);
  uint32_t *patch = reinterpret_cast<uint32_t *>(smem + kWeightU4 * 16);
  uint32_t *pool = patch + kPatchWords;
  int4 *koff = reinterpret_cast<int4 *>(pool + kPH * kPW * kPoolPitch);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.z, py0 = blockIdx.y * kPH, px0 = blockIdx.x * kPW;
  bool ovf = false;

  for (int i = tid; i < kWeightU4; i += kThreads) wsm[i] = __ldg(p.packed + i);
  for (int i = tid; i < kPH * kPW * kPoolPitch; i += kThreads) pool[i] = 0u;  // +0.0f
  if (tid < kSteps * 4) {  // k = 16 s + 2 t + {0, 1, 8, 9}: patch offset of (c, ky, kx); padding k reads word 0 (weight 0)
    const int s = tid >> 2, t = tid & 3;
    int o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = 16 * s + 2 * t + (j & 1) + (j >> 1) * 8;
      const int c = k / 49, r = k % 49;
      o[j] = k < kKReal ? (c * kIR + r / 7) * kIP + r % 7 : 0;
    }
    koff[tid] = make_int4(o[0], o[1], o[2], o[3]);
  }
  // input patch: rows 4 py0 - 5 + [0, 39), columns 4 px0 - 5 + [0, 71); zero outside the image (the conv's padding)
  const int iy0 = 4 * py0 - 5, ix0 = 4 * px0 - 5;
  const float *img = p.in + static_cast<size_t>(b) * kCin * p.H * p.W;
  for (int i = tid; i < kCin * kIR * kIC; i += kThreads) {
    const int c = i / (kIR * kIC), r = (i / kIC) % kIR, col = i % kIC;
    const int iy = iy0 + r, ix = ix0 + col;
    const float v = (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) ? __ldg(img + (static_cast<size_t>(c) * p.H + iy) * p.W + ix) : 0.f;
    patch[(c * kIR + r) * kIP + col] = pair_word(v, ovf);
  }
  __syncthreads();

  const int g = lane >> 2, t = lane & 3;
  const int cy0 = 2 * py0 - 1, cx0 = 2 * px0 - 1;  // conv coordinates of the tile's conv pixel 0
  for (int mt = warp; mt < kMTiles; mt += kWarps) {
    const int m0 = mt * 16 + g, m1 = m0 + 8;
    const int a0 = min(m0, kConvPx - 1), a1 = min(m1, kConvPx - 1);
    const uint32_t *base0 = patch + 2 * (a0 / kCC) * kIP + 2 * (a0 % kCC);
    const uint32_t *base1 = patch + 2 * (a1 / kCC) * kIP + 2 * (a1 % kCC);
    float hh[8][4], ll[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) hh[j][e] = ll[j][e] = 0.f;
#pragma unroll 1
    for (int s = 0; s < kSteps; ++s) {
      const int4 o = koff[s * 4 + t];
      const uint32_t r00 = base0[o.x], r01 = base0[o.y], r02 = base0[o.z], r03 = base0[o.w];
      const uint32_t r10 = base1[o.x], r11 = base1[o.y], r12 = base1[o.z], r13 = base1[o.w];
      const uint4 ahi = make_uint4(__byte_perm(r00, r01, 0x5410), __byte_perm(r10, r11, 0x5410), __byte_perm(r02, r03, 0x5410),
                                   __byte_perm(r12, r13, 0x5410));
      const uint4 alo = make_uint4(__byte_perm(r00, r01, 0x7632), __byte_perm(r10, r11, 0x7632), __byte_perm(r02, r03, 0x7632),
                                   __byte_perm(r12, r13, 0x7632));
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint4 w = wsm[(s * 8 + j) * 32 + lane];
        tc::mma16816(hh[j], ahi, w.x, w.y);
        tc::mma16816(ll[j], ahi, w.z, w.w);
        tc::mma16816(ll[j], alo, w.x, w.y);
      }
    }
    // epilogue: rows m0 (elements 0, 1) and m1 (2, 3), channels 8 j + 2 t + (e & 1)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = h ? m1 : m0;
      if (m >= kConvPx) continue;
      const int r = m / kCC, c = m % kCC;
      const int cy = cy0 + r, cx = cx0 + c;
      if (cy < 0 || cy >= p.cH || cx < 0 || cx >= p.cW) continue;  // MaxPool's padding
      // pooled local rows whose window {2 i, 2 i + 1, 2 i + 2} holds r, the same for columns
      const int ri = r >> 1, ci = c >> 1;
      const bool r2 = !(r & 1) && ri > 0 && ri < kPH, c2 = !(c & 1) && ci > 0 && ci < kPW;
      const int rA = ri < kPH ? ri : ri - 1, cA = ci < kPW ? ci : ci - 1;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int n = 8 * j + 2 * t + e;
          const float v = fmaf(fmaf(ll[j][2 * h + e], kLoInv, hh[j][2 * h + e]), __ldg(p.scale + n), __ldg(p.shift + n));
          const uint32_t bits = __float_as_uint(v > 0.f ? v : 0.f);
          atomicMax(pool + (rA * kPW + cA) * kPoolPitch + n, bits);
          if (c2) atomicMax(pool + (rA * kPW + cA - 1) * kPoolPitch + n, bits);
          if (r2) atomicMax(pool + ((rA - 1) * kPW + cA) * kPoolPitch + n, bits);
          if (r2 && c2) atomicMax(pool + ((rA - 1) * kPW + cA - 1) * kPoolPitch + n, bits);
        }
    }
  }
  __syncthreads();
  // pooled tile -> pixel rows: one thread per (cell, 8 channels)
  for (int i = tid; i < kPH * kPW * (kCout / 8); i += kThreads) {
    const int cell = i >> 3, q = i & 7;
    const int py = py0 + cell / kPW, px = px0 + cell % kPW;
    if (py >= p.pH || px >= p.pW) continue;
    const uint32_t *src = pool + cell * kPoolPitch + 8 * q;
    uint4 hi, lo;
    __half2 *h2 = reinterpret_cast<__half2 *>(&hi), *l2 = reinterpret_cast<__half2 *>(&lo);
#pragma unroll
    for (int k = 0; k < 4; ++k) split_h16x2(__uint_as_float(src[2 * k]), __uint_as_float(src[2 * k + 1]), h2[k], l2[k], ovf);
    uint8_t *o = p.out + ((static_cast<size_t>(b) * p.pH + py) * p.pW + px) * (4 * kCout) + (q >> 2) * 128 + (q & 3) * 16;
    *reinterpret_cast<uint4 *>(o) = hi;
    *reinterpret_cast<uint4 *>(o + 64) = lo;
  }
  if (ovf && p.status) atomicOr(p.status, 1);
}

// W [64][3][7][7] fp32 -> [kSteps][8 n-tiles][32 lanes] x (hi b0, hi b1, lo' b0, lo' b1): lane (g, t) of n-tile j holds
// W[8 j + g][k] for k = 16 s + 2 t + {0, 1} (b0) and + {8, 9} (b1), low half first; k >= 147 zero
__global__ void resnet_stem_pack_kernel(const float *__restrict__ w, uint4 *__restrict__ packed, int32_t *status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= kWeightU4) return;
  const int lane = i & 31, j = (i >> 5) & 7, s = i >> 8;
  const int n = 8 * j + (lane >> 2), t = lane & 3;
  bool ovf = false;
  uint32_t hi[2], lo[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int k = 16 * s + 2 * t + 8 * r;
    const float x0 = k < kKReal ? w[n * kKReal + k] : 0.f, x1 = k + 1 < kKReal ? w[n * kKReal + k + 1] : 0.f;
    __half2 h, l;
    split_h16x2(x0, x1, h, l, ovf);
    hi[r] = *reinterpret_cast<uint32_t *>(&h);
    lo[r] = *reinterpret_cast<uint32_t *>(&l);
  }
  packed[i] = make_uint4(hi[0], hi[1], lo[0], lo[1]);
  if (ovf && status) atomicOr(status, 1);
}

}  // namespace stem
}  // namespace p3d

using namespace p3d;

extern "C" size_t p3d_resnet_stem_packed_weight_bytes(void) { return static_cast<size_t>(stem::kWeightU4) * 16; }

extern "C" int p3d_resnet_stem_pack_weights(const float *weight, void *packed, int32_t *status_dev, p3d_stream_t stream) {
  if (!weight || !packed || (reinterpret_cast<uintptr_t>(packed) & 15)) return P3D_ERR_INVALID_ARG;
  stem::resnet_stem_pack_kernel<<<div_up(stem::kWeightU4, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      weight, static_cast<uint4 *>(packed), status_dev);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" int p3d_resnet_stem_h16(const float *in, int B, int H, int W, const void *packed_weight, const float *scale,
                                   const float *shift, void *out_h16, int32_t *status_dev, p3d_stream_t stream) {
  if (!in || !packed_weight || !scale || !shift || !out_h16 || B < 1 || H < 1 || W < 1 ||
      (reinterpret_cast<uintptr_t>(packed_weight) & 15) || (reinterpret_cast<uintptr_t>(out_h16) & 15))
    return P3D_ERR_INVALID_ARG;
  stem::Params p;
  p.in = in;
  p.packed = static_cast<const uint4 *>(packed_weight);
  p.scale = scale;
  p.shift = shift;
  p.out = static_cast<uint8_t *>(out_h16);
  p.B = B;
  p.H = H;
  p.W = W;
  p.cH = (H - 1) / 2 + 1;  // (H + 6 - 7) / 2 + 1
  p.cW = (W - 1) / 2 + 1;
  p.pH = (p.cH - 1) / 2 + 1;  // (cH + 2 - 3) / 2 + 1
  p.pW = (p.cW - 1) / 2 + 1;
  p.status = status_dev;
  if (B > 65535 || static_cast<long long>(B) * 3 * H * W > 0x7fffffffll) return P3D_ERR_UNSUPPORTED;
  const dim3 grid(div_up(p.pW, stem::kPW), div_up(p.pH, stem::kPH), B);
  if (grid.y > 65535) return P3D_ERR_UNSUPPORTED;
  P3D_CUDA_CHECK(cudaFuncSetAttribute(stem::resnet_stem_h16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(stem::kSmemBytes)));
  stem::resnet_stem_h16_kernel<<<grid, stem::kThreads, stem::kSmemBytes, static_cast<cudaStream_t>(stream)>>>(p);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
