// Dense 2-D convolution on wgmma (tf32) for the RPN / neck / CenterHead row (SURVEY.md §8f-1; reference:
// backbones/second_backbone.py:72-120, necks/second_fpn.py:99-160, detection/centerpoint/center_head.py:43-220).
// Kept for models whose activations leave fp16's range; the default dense path is dense_conv_f16.cu.
//
// The image is kept as "pixel split rows" [B*H*W][2][C] (NHWC with the tf32 hi half of all channels, then the lo half —
// the row format of the sparse-conv layers with row = pixel), so a 3x3 tap of 32 input channels for a 16 x 8 pixel
// tile is one 4-D TMA box {32 ch, 16 x, 8 y, 1 b} at the shifted coordinate: zero padding is the tensor map's
// out-of-bounds fill, a stride-2 conv is the map's element stride, and the box lands in shared memory as the
// SWIZZLE_128B K-major operand tile (128 rows x 128 B).  3xTF32: A_hi x B_hi into one register accumulator (one tap's
// partial, added to an fp32 register total with round-to-nearest FADDs after the tap's last channel group: the tensor
// core's own accumulation drifts over a whole 9 x Cin / 8 k-step chain), A_lo x B_hi + A_hi x B_lo into a second
// (warpgroup g: rows 64g .. 64g+63 of the tile), weights of the use by cp.async.bulk,
// BN/bias/ReLU epilogue writing split rows (at a column offset: channel concat for free) or fp32 NCHW planes (the head
// outputs centerpoint_postprocess reads).
//
//   work item   (batch, 16 x 8 output tile, N tile of the output channels[, tap of a k = s transposed conv])
//   step        one (tap, 32-channel group) of an item: image tile (hi, lo) + weight slice in one ring slot.  Thread 0
//               keeps the ring STAGES - 1 steps ahead across work items (TMA, mbarrier complete_tx); all 256 threads
//               issue the wgmma of their warpgroup and run its epilogue.
#include <cuda.h>

#include "p3d_b200.h"
#include "tc_common.cuh"

namespace p3d {
namespace dc {

using namespace tc;

constexpr int kTW = 16, kTH = 8;  // output tile: 16 x 8 pixels = the 128 rows of one CTA tile
static_assert(kTW * kTH == kM, "tile must have 128 pixels");

struct Params {
  int B, H, W, Cin;          // input image (pixel split rows [B*H*W][2][Cin])
  int taps, kw, stride, pad;  // conv geometry (taps = kh * kw); transposed conv: taps = up * up, stride = pad = 0 here
  int up;                    // 1 = convolution; > 1 = transposed conv with kernel = stride = up
  int oH, oW;                // extent of the tiled grid (conv: output image; transposed: input image)
  int tiles_x, tiles_y, n_ntiles;
  int cout;                  // valid output channels (N tiles are zero-padded above it)
  int out_H, out_W;          // output image
  int out_C, out_c0;         // split-row output: channels per row and first column written by this layer
  int relu;
};

template <int N>
struct Cfg {
  static constexpr int KC = 32;
  static constexpr int A_TILE = KC * kM * 4;
  static constexpr int A_STAGE = 2 * A_TILE;
  static constexpr int B_STAGE = 2 * KC * N * 4;
  static constexpr int STAGE = A_STAGE + B_STAGE;
  static constexpr int MIN_CTAS = (N <= 64) ? 2 : 1;
  static constexpr int BUDGET = (N <= 64) ? 100 * 1024 : 192 * 1024;
  static constexpr int S_RAW = BUDGET / STAGE;
  static constexpr int STAGES = S_RAW > 8 ? 8 : (S_RAW < 2 ? 2 : S_RAW);
  static constexpr int ACC = N / 2;
  static_assert(N % 16 == 0 && N >= 16 && N <= 128, "N tile: 16 .. 128 in steps of 16");
  static_assert(STAGE % 1024 == 0, "SWIZZLE_128B tiles need 1024-byte alignment");
};

__device__ __forceinline__ void tma_tile4d(uint32_t dst, const CUtensorMap *map, int c, int x, int y, int b, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];" ::
          "r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c), "r"(x), "r"(y), "r"(b), "r"(bar)
      : "memory");
}

struct Item {
  int nt, tap0, tx0, ty0, b;
};
// N tile fastest (neighbouring CTAs share the image tile in L2), then tap (transposed conv), x, y, batch
__device__ __forceinline__ Item decode(long long w, const Params &p) {
  Item it;
  long long q = w;
  it.nt = static_cast<int>(q % p.n_ntiles);
  q /= p.n_ntiles;
  it.tap0 = 0;
  if (p.up > 1) {
    it.tap0 = static_cast<int>(q % (p.up * p.up));
    q /= p.up * p.up;
  }
  it.tx0 = static_cast<int>(q % p.tiles_x) * kTW;
  q /= p.tiles_x;
  it.ty0 = static_cast<int>(q % p.tiles_y) * kTH;
  it.b = static_cast<int>(q / p.tiles_y);
  return it;
}

template <int N>
__global__ void __launch_bounds__(kThreads, Cfg<N>::MIN_CTAS)
    dense_conv_kernel(const __grid_constant__ CUtensorMap in_map, const Params p, const float *__restrict__ packed_w,
                      const float *__restrict__ scale, const float *__restrict__ shift, float *__restrict__ out_split,
                      float *__restrict__ out_nchw) {
  using C = Cfg<N>;
  constexpr int S = C::STAGES;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");  // the input image is the previous layer's output
  const int up2 = p.up * p.up;
  const long long n_work = static_cast<long long>(p.B) * p.tiles_y * p.tiles_x * p.n_ntiles * (p.up > 1 ? up2 : 1);
  if (static_cast<long long>(blockIdx.x) >= n_work) return;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) unsigned long long s_full[8];

  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127;
  if (tid == 0) {
    for (int s = 0; s < S; ++s) mbar_init(smem_u32(&s_full[s]), 1);  // the TMA lane's expect_tx arrival (rows + weights)
    fence_mbar_init();
  }
  const uint32_t ring = smem_u32(smem);
  const int G = p.Cin / C::KC;
  const int n_uses = (p.up > 1 ? 1 : p.taps) * G;  // steps per item
  const long long n_items = (n_work - blockIdx.x + gridDim.x - 1) / gridDim.x;
  const long long n_steps = n_items * n_uses;

  // thread 0: loads of global step q (item q / n_uses of this CTA) into slot q % S
  auto issue = [&](long long q) {
    const Item im = decode(blockIdx.x + (q / n_uses) * gridDim.x, p);
    const int u = static_cast<int>(q % n_uses);
    const int t = (p.up > 1 ? im.tap0 : u / G), g = u % G;
    const int dy = p.up > 1 ? 0 : t / p.kw, dx = p.up > 1 ? 0 : t % p.kw;
    const int x = im.tx0 * p.stride - p.pad + dx, y = im.ty0 * p.stride - p.pad + dy;  // may be negative: zero fill
    const uint32_t slot = static_cast<uint32_t>(q % S);
    const uint32_t st = ring + slot * C::STAGE, bar = smem_u32(&s_full[slot]);
    const float *w_tile = packed_w + static_cast<size_t>(im.nt) * p.taps * p.Cin * (2 * N);
    mbar_arrive_expect_tx(bar, static_cast<uint32_t>(C::STAGE));
    tma_tile4d(st, &in_map, g * C::KC, x, y, im.b, bar);                       // hi half of the 32 channels
    tma_tile4d(st + C::A_TILE, &in_map, p.Cin + g * C::KC, x, y, im.b, bar);   // lo half
    bulk_g2s(st + C::A_STAGE, w_tile + (static_cast<size_t>(t) * p.Cin + g * C::KC) * (2 * N),
             static_cast<uint32_t>(C::B_STAGE), bar);
  };
  long long next = 0;  // thread 0: next step to load
  float acc[C::ACC], accx[C::ACC], tot[C::ACC];  // hi x hi of the current tap | cross terms | hi x hi of done taps
  long long q = 0;
  for (long long w = blockIdx.x; w < n_work; w += gridDim.x) {
    const Item im = decode(w, p);
#pragma unroll
    for (int i = 0; i < C::ACC; ++i) acc[i] = accx[i] = tot[i] = 0.f;
    for (int u = 0; u < n_uses; ++u, ++q) {
      __syncthreads();  // the wgmma of step q - 1 have retired in both warpgroups: its slot is free
      if (tid == 0)
        for (; next < n_steps && next <= q + S - 1; ++next) issue(next);
      const uint32_t slot = static_cast<uint32_t>(q % S);
      mbar_wait(smem_u32(&s_full[slot]), static_cast<uint32_t>((q / S) & 1));
      const uint32_t a_hi = ring + slot * C::STAGE + static_cast<uint32_t>(wg * 64 * 128), a_lo = a_hi + C::A_TILE;
      const uint32_t b_hi = ring + slot * C::STAGE + C::A_STAGE, b_lo = b_hi + N * 16;  // rows 0..N-1 = hi, N..2N-1 = lo
      const uint32_t tap_first = (u % G) == 0;  // the tap's hi x hi partial starts over (scale_d = 0)
      wg_fence();
#pragma unroll
      for (int j = 0; j < C::KC / 8; ++j) {
        const uint32_t bo = static_cast<uint32_t>(2 * j) * (2 * N * 16);
        const uint64_t dah = desc_sw128(a_hi + j * 32), dal = desc_sw128(a_lo + j * 32);
        const uint64_t dbh = smem_desc(b_hi + bo, 2 * N * 16, 128), dbl = smem_desc(b_lo + bo, 2 * N * 16, 128);
        wg::mma_tf32<N>(accx, dal, dbh, 1u);
        wg::mma_tf32<N>(accx, dah, dbl, 1u);
        wg::mma_tf32<N>(acc, dah, dbh, (tap_first && j == 0) ? 0u : 1u);
      }
      wg_commit();
      wg_wait<0>();
      if (u % G == G - 1) {  // last channel group of the tap: its partial joins the total
        wg_fence_acc<C::ACC>(acc);
#pragma unroll
        for (int i = 0; i < C::ACC; ++i) tot[i] += acc[i];
      }
    }
    wg_fence_acc<C::ACC>(accx);

    // ---------------------------------------------------------------- epilogue (accumulator fragment)
#pragma unroll
    for (int i = 0; i < C::ACC; i += 2) {
      const int m = wg * 64 + frag_row(i, wtid), c = frag_col(i, wtid);  // tile pixel, N-tile column
      const int iy = im.ty0 + m / kTW, ix = im.tx0 + m % kTW;
      const int ch = im.nt * N + c;  // output channel
      if (iy >= p.oH || ix >= p.oW || ch >= p.cout) continue;
      const int Y = iy * p.up + (p.up > 1 ? im.tap0 / p.up : 0), X = ix * p.up + (p.up > 1 ? im.tap0 % p.up : 0);
      const size_t orow = (static_cast<size_t>(im.b) * p.out_H + Y) * p.out_W + X;
      float o[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float v = accx[i + e] + tot[i + e];
        if (ch + e < p.cout) {
          if (scale) v = v * __ldg(scale + ch + e);
          if (shift) v = v + __ldg(shift + ch + e);
        }
        if (p.relu) v = fmaxf(v, 0.f);
        o[e] = v;
      }
      if (out_split) {  // channel counts of split-row layers are multiples of 16: whole pairs
        float h[2], l[2];
        split_tf32(o[0], h[0], l[0]);
        split_tf32(o[1], h[1], l[1]);
        float *oh = out_split + orow * (2 * static_cast<size_t>(p.out_C)) + p.out_c0 + ch;
        *reinterpret_cast<float2 *>(oh) = make_float2(h[0], h[1]);
        *reinterpret_cast<float2 *>(oh + p.out_C) = make_float2(l[0], l[1]);
      }
      if (out_nchw) {  // fp32 planes [B, cout, out_H, out_W]
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (ch + e < p.cout) out_nchw[((static_cast<size_t>(im.b) * p.cout + ch + e) * p.out_H + Y) * p.out_W + X] = o[e];
      }
    }
  }
}

// fp32 NCHW image -> pixel split rows [B*H*W][2][C] (32 x 32 tile transpose through shared memory)
__global__ void __launch_bounds__(256) nchw_to_pixel_split_kernel(const float *__restrict__ in, int C, long long HW,
                                                                  float *__restrict__ out) {
  __shared__ float s_t[32][33];
  const int b = blockIdx.z;
  const long long p0 = static_cast<long long>(blockIdx.x) * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int k = ty; k < 32; k += 8) {
    const int c = c0 + k;
    const long long px = p0 + tx;
    s_t[k][tx] = (c < C && px < HW) ? in[(static_cast<size_t>(b) * C + c) * HW + px] : 0.f;
  }
  __syncthreads();
  for (int k = ty; k < 32; k += 8) {
    const long long px = p0 + k;
    const int c = c0 + tx;
    if (c < C && px < HW) {
      float h, l;
      split_tf32(s_t[tx][k], h, l);
      float *row = out + (static_cast<size_t>(b) * HW + px) * (2 * static_cast<size_t>(C));
      row[c] = h;
      row[C + c] = l;
    }
  }
}

inline int make_image_map(const float *img, int B, int H, int W, int Cin, int stride, CUtensorMap *map) {
  using Encode = CUresult (*)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                              const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static Encode encode = nullptr;
  if (!encode) {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) != cudaSuccess || !fn)
      return P3D_ERR_UNSUPPORTED;
    encode = reinterpret_cast<Encode>(fn);
  }
  const cuuint64_t row = static_cast<cuuint64_t>(2 * Cin) * sizeof(float);
  const cuuint64_t gdim[4] = {static_cast<cuuint64_t>(2 * Cin), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H),
                              static_cast<cuuint64_t>(B)};
  const cuuint64_t gstride[3] = {row, row * W, row * W * H};
  // with an element stride s the box extent is s x the number of elements loaded (cuda.h, cuTensorMapEncodeTiled)
  const cuuint32_t box[4] = {32u, static_cast<cuuint32_t>(kTW * stride), static_cast<cuuint32_t>(kTH * stride), 1u};
  const cuuint32_t estride[4] = {1u, static_cast<cuuint32_t>(stride), static_cast<cuuint32_t>(stride), 1u};
  const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float *>(img), gdim, gstride, box, estride,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? P3D_OK : P3D_ERR_INVALID_ARG;
}

template <int N>
int launch(const CUtensorMap &map, const Params &p, const float *packed, const float *scale, const float *shift,
           float *out_split, float *out_nchw, cudaStream_t st) {
  using C = Cfg<N>;
  const size_t smem = static_cast<size_t>(C::STAGES) * C::STAGE + 1024;
  auto kern = dense_conv_kernel<N>;
  P3D_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  const long long work = static_cast<long long>(p.B) * p.tiles_y * p.tiles_x * p.n_ntiles * (p.up > 1 ? p.up * p.up : 1);
  const long long slots = static_cast<long long>(num_sms()) * C::MIN_CTAS;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned int>(work < slots ? work : slots));
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  P3D_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, map, p, packed, scale, shift, out_split, out_nchw));
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

}  // namespace dc
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_nchw_to_pixel_split(const float *in, int B, int C, int H, int W, float *out_split,
                                       p3d_stream_t stream) {
  if (!in || !out_split || B < 1 || C < 1 || H < 1 || W < 1) return P3D_ERR_INVALID_ARG;
  const long long hw = static_cast<long long>(H) * W;
  dim3 grid(static_cast<unsigned int>((hw + 31) / 32), static_cast<unsigned int>((C + 31) / 32), B);
  dc::nchw_to_pixel_split_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(in, C, hw, out_split);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" size_t p3d_dense_conv2d_packed_weight_bytes(int taps, int Cin, int Cout, int n_tile) {
  if (taps < 1 || Cin < 32 || Cin % 32 || Cout < 1 || (n_tile != 16 && n_tile != 64 && n_tile != 128)) return 0;
  const size_t tiles = static_cast<size_t>((Cout + n_tile - 1) / n_tile);
  return align_up(tiles * taps * Cin * (2 * static_cast<size_t>(n_tile)) * sizeof(float));
}

extern "C" int p3d_dense_conv2d_split(const float *in_split, int B, int H, int W, int Cin, const float *packed_weight,
                                      int Cout, int n_tile, int kh, int kw, int stride, int pad, int up,
                                      const float *scale, const float *shift, int relu, float *out_split, int out_C,
                                      int out_c0, float *out_nchw, p3d_stream_t stream) {
  if (!in_split || !packed_weight || (!out_split && !out_nchw) || B < 1 || H < 1 || W < 1 || Cout < 1)
    return P3D_ERR_INVALID_ARG;
  if (Cin < 32 || Cin % 32 || (n_tile != 16 && n_tile != 64 && n_tile != 128)) return P3D_ERR_UNSUPPORTED;
  if (up < 1 || (up > 1 && (kh != up || kw != up || stride != up || pad != 0))) return P3D_ERR_UNSUPPORTED;
  if (up == 1 && (kh < 1 || kw < 1 || kh * kw > 32 || stride < 1 || stride > 2 || pad < 0)) return P3D_ERR_UNSUPPORTED;
  if (out_split && (Cout % 16 || out_C % 4 || out_c0 % 4 || out_c0 + Cout > out_C)) return P3D_ERR_INVALID_ARG;
  if ((reinterpret_cast<uintptr_t>(in_split) & 15) || (reinterpret_cast<uintptr_t>(packed_weight) & 15) ||
      (reinterpret_cast<uintptr_t>(out_split) & 15))
    return P3D_ERR_INVALID_ARG;
  dc::Params p;
  p.B = B;
  p.H = H;
  p.W = W;
  p.Cin = Cin;
  p.taps = kh * kw;
  p.kw = kw;
  p.up = up;
  p.stride = up > 1 ? 1 : stride;
  p.pad = up > 1 ? 0 : pad;
  p.oH = up > 1 ? H : (H + 2 * pad - kh) / stride + 1;
  p.oW = up > 1 ? W : (W + 2 * pad - kw) / stride + 1;
  if (p.oH < 1 || p.oW < 1) return P3D_ERR_INVALID_ARG;
  p.out_H = up > 1 ? H * up : p.oH;
  p.out_W = up > 1 ? W * up : p.oW;
  p.tiles_x = (p.oW + dc::kTW - 1) / dc::kTW;
  p.tiles_y = (p.oH + dc::kTH - 1) / dc::kTH;
  p.n_ntiles = (Cout + n_tile - 1) / n_tile;
  p.cout = Cout;
  p.out_C = out_C;
  p.out_c0 = out_c0;
  p.relu = relu;
  CUtensorMap map;
  const int rc = dc::make_image_map(in_split, B, H, W, Cin, p.stride, &map);
  if (rc != P3D_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (n_tile == 16) return dc::launch<16>(map, p, packed_weight, scale, shift, out_split, out_nchw, st);
  if (n_tile == 64) return dc::launch<64>(map, p, packed_weight, scale, shift, out_split, out_nchw, st);
  return dc::launch<128>(map, p, packed_weight, scale, shift, out_split, out_nchw, st);
}
