// The fp16-pair ("H16") value format, the activation format between all tensor-core layers (DESIGN.md §2):
// x = hi + lo' * 2^-11 with hi = fp16(x), lo' = fp16((x - hi) * 2^11).  Both halves carry 11 significant bits, and the
// power-of-two scale keeps lo' in fp16's normal range, so a pair holds 22 mantissa bits.  Values with |x| > 65504 are
// saturated and raise the caller's overflow flag (status bit 0 of the kernels).
#pragma once
#include <cuda_fp16.h>

#include <cstdint>

namespace p3d {

constexpr float kLoScale = 2048.0f, kLoInv = 1.0f / 2048.0f;

// x -> (hi, lo') fp16 pair; sets ovf when |x| leaves fp16's range (value saturated)
__device__ __forceinline__ void split_h16(float x, __half &hi, __half &lo, bool &ovf) {
  if (fabsf(x) > 65504.0f) {
    ovf = true;
    x = copysignf(65504.0f, x);
  }
  hi = __float2half_rn(x);
  lo = __float2half_rn((x - __half2float(hi)) * kLoScale);
}

// split_h16 of two values with paired conversions (round to nearest either way: the same bits)
__device__ __forceinline__ void split_h16x2(float a, float b, __half2 &hi, __half2 &lo, bool &ovf) {
  if (fabsf(a) > 65504.0f) {
    ovf = true;
    a = copysignf(65504.0f, a);
  }
  if (fabsf(b) > 65504.0f) {
    ovf = true;
    b = copysignf(65504.0f, b);
  }
  hi = __floats2half2_rn(a, b);
  const float2 h = __half22float2(hi);
  lo = __floats2half2_rn((a - h.x) * kLoScale, (b - h.y) * kLoScale);
}

__device__ __forceinline__ float merge_h16(__half hi, __half lo) { return fmaf(__half2float(lo), kLoInv, __half2float(hi)); }

// channels 8 q .. 8 q + 7 of a pixel row, merged to fp32: hi at (q / 4) * 128 + (q % 4) * 16, lo' 64 bytes further
__device__ __forceinline__ void load8(const uint8_t *px, int q, float v[8]) {
  const uint8_t *g = px + (q >> 2) * 128 + (q & 3) * 16;
  const uint4 hi = __ldg(reinterpret_cast<const uint4 *>(g)), lo = __ldg(reinterpret_cast<const uint4 *>(g + 64));
  const __half2 *h2 = reinterpret_cast<const __half2 *>(&hi), *l2 = reinterpret_cast<const __half2 *>(&lo);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 fh = __half22float2(h2[k]), fl = __half22float2(l2[k]);
    v[2 * k] = fmaf(fl.x, kLoInv, fh.x);
    v[2 * k + 1] = fmaf(fl.y, kLoInv, fh.y);
  }
}

}  // namespace p3d
