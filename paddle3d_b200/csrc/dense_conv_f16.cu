// Dense 2-D convolution on wgmma with fp16 (hi, lo') pair operands for the RPN / neck / CenterHead row (SURVEY.md §8f-1;
// reference: backbones/second_backbone.py:72-120, necks/second_fpn.py:99-160, detection/centerpoint/center_head.py:43-220).
//
// Images travel between layers as "pixel H16 rows": NHWC, each pixel's C channels as groups of 32 channels
// [hi 32 halfs | lo' 32 halfs] (128 bytes per group; x = hi + lo' * 2^-11, the sparse layers' row format with row = pixel).
// One (32-channel group) x (pixel box) TMA load therefore lands in shared memory as a SWIZZLE_128B K-major operand tile
// whose k-steps 0,1 are the hi halves and 2,3 the lo' halves; the three partial products run as
//   D[0, N) += A_hi x B_hi          D[N, 2N) += A_hi x B_lo' + A_lo' x B_hi        out = D[0, N) + D[N, 2N) * 2^-11
// (three m64nN wgmma per 16-channel k-step and warpgroup; the accumulators live in registers).
//
//   * HALO mode (3x3, stride 1, pad 1): the haloed tile (10 x 18 pixels for an 8 x 16 output tile, or 10 x 34 for
//     8 x 32 = two M tiles) of a 32-channel group is loaded ONCE; the A operand of tap (dy, dx) is the same
//     shared-memory tile read through a descriptor whose start address is shifted by (dy * 10 + dx) rows and whose 8-row
//     group stride (SBO) is one haloed image row (1280 bytes).  The swizzle is a function of the absolute shared-memory
//     address bits, so TMA's writes and the shifted wgmma reads agree (descriptor base_offset 0, tests/test_gpu_dense.py).
//   * TAP mode (1x1, stride 2, transposed k = s): one TMA box per (tap, group).
//   * MT = 2 (N tile <= 64): two M tiles (8 x 32 pixels) share every weight block: half the weight traffic per flop.
//
//   work item   (batch, pixel tile, N tile[, tap of a k = s transposed conv]), N tile fastest
//   step        (A unit, tap): HALO one A unit per 32-channel group serves 9 steps, TAP one A unit per step.  Thread 0
//               keeps an activation ring (NA) and a weight ring (NB) ahead of the consumers across work items (TMA /
//               cp.async.bulk, mbarrier complete_tx); warpgroup g computes rows 64g .. 64g+63 of every M tile and runs
//               their epilogue from its registers.
#include <cuda.h>
#include <cuda_fp16.h>

#include "p3d_b200.h"
#include "tc_common.cuh"

namespace p3d {
namespace dcf {

using namespace tc;

constexpr int kTW = 8, kTH = 16;        // output tile of one M = 128 tile: 8 x 16 pixels
constexpr int kMaxA = 6, kMaxB = 12;    // activation / weight ring depth limits
constexpr float kLoScale = 2048.0f, kLoInv = 1.0f / 2048.0f;

struct Params {
  int B, H, W, Cin;           // input image (pixel H16 rows [B*H*W][4 * Cin bytes])
  int taps, kw, stride, pad;  // conv geometry (taps = kh * kw); transposed conv: taps = up * up
  int up;                     // 1 = convolution; > 1 = transposed conv with kernel = stride = up
  int oH, oW;                 // extent of the tiled grid (conv: output image; transposed: input image)
  int tiles_x, tiles_y, n_ntiles;
  int cout;                   // valid output channels (N tiles are zero-padded above it)
  int out_H, out_W;           // output image
  int out_C, out_c0;          // H16 output: channels per row and first channel written by this layer
  int relu;
  const uint8_t *packed_w;    // [n_ntiles][taps][Cin / 16] k-blocks of 64 * N bytes
  const float *scale, *shift;
  uint8_t *out_h16;           // or null
  float *out_nchw;            // fp32 planes [B, cout, out_H, out_W] or null
  int32_t *status;            // bit 0: fp16 range overflow while writing out_h16
  // grouped mode (the 36 output convs of the CenterHead as ONE launch): N tile nt reads input channels
  // [nt * Cin, (nt + 1) * Cin) of an image with in_C channels, uses weight tile nt, and writes its first grp_cnt[nt]
  // columns to the fp32 planes grp_plane0[nt] .. of out_nchw ([B, cout planes, out_H, out_W]); shift is [n_ntiles][N]
  int grouped, in_C;
  const int32_t *grp_plane0, *grp_cnt;
  int base_offset_mode;       // 0 (default): base_offset field zero; 1: address bits 7-9 of the shifted start address
  int w_bytes;                // weight-stationary kernel: bytes of one N tile's weight image (taps * Cin / 16 k-blocks)
};

// PITCH: pixels per row of the haloed tile in shared memory: 10 (tight: 8 + 2) or 16 (8-row groups stay 1024-byte aligned)
// WS ("weight-stationary", HALO only): the whole weight image of an N tile (taps * Cin / 16 k-blocks, <= 144 KB) stays in
// shared memory while the CTA walks a contiguous range of pixel tiles of that N tile; only the haloed activation tiles
// stream.  For layers with few input and many output channels (the 64 -> 36 x 64 ConvModules of the CenterHead) this
// replaces 43 B/clk of weight ingest per SM - the L2 -> SM limit - by 13 B/clk of activations.
template <int N, int MT, bool HALO, int PITCH, bool WS = false>
struct Cfg {
  static constexpr int A_ROWS = HALO ? PITCH * (kTH * MT + 2) : kM * MT;     // rows of 128 bytes per activation buffer
  static constexpr int A_BYTES = ((A_ROWS * 128 + 1023) / 1024) * 1024;
  static constexpr int B_BYTES = 128 * N;                                    // weight blocks of one (tap, group): 2 k-blocks
  static constexpr int B_BLK = 64 * N;
  // TAP mode: every step needs a new activation buffer, so both rings get the same depth; HALO: 2 (WS: 3) buffers
  static constexpr int NA_TAP_RAW = (227 - 6) * 1024 / (A_BYTES + B_BYTES);
  static constexpr int NA = WS ? 3 : (HALO ? 2 : (NA_TAP_RAW > kMaxA ? kMaxA : NA_TAP_RAW));
  static constexpr int BUDGET = (227 - 6) * 1024 - NA * A_BYTES;  // 227 KB - alignment slack - static (barriers)
  static constexpr int NB_RAW = BUDGET / B_BYTES;
  static constexpr int NB = NB_RAW > kMaxB ? kMaxB : NB_RAW;                 // weight ring depth
  static constexpr int ACC = MT * N;                                         // fp32 registers per thread
  static constexpr int SPU = HALO ? 9 : 1;                                   // steps per activation buffer
  static_assert(N == 16 || N == 64 || N == 128, "N tile: 16 (grouped output convs), 64 or 128");
  static_assert(MT == 1 || MT == 2, "one or two M tiles");
  static_assert(MT * N <= 128, "accumulators: at most 128 registers per thread");
  static_assert(WS || NB >= 3, "weight ring too shallow");
  static_assert(NA >= 2 && NA <= kMaxA, "activation ring depth");
  static_assert(!WS || (HALO && MT == 1), "weight-stationary: haloed 3x3 tiles, one M tile");
};

__device__ __forceinline__ void tma_tile4d(uint32_t dst, const CUtensorMap *map, int c, int x, int y, int b, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];" ::
          "r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c), "r"(x), "r"(y), "r"(b), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void split_h16(float x, __half &hi, __half &lo, bool &ovf) {
  if (fabsf(x) > 65504.0f) {
    ovf = true;
    x = copysignf(65504.0f, x);
  }
  hi = __float2half_rn(x);
  lo = __float2half_rn((x - __half2float(hi)) * kLoScale);
}

struct Item {
  int nt, tap0, tx0, ty0, b;
};
template <bool WS = false>
__device__ __forceinline__ Item decode(long long w, const Params &p, int th) {
  Item it;
  long long q = w;
  if (WS) {  // N tile slowest: a CTA's contiguous item range stays on one N tile
    const long long pix = static_cast<long long>(p.B) * p.tiles_y * p.tiles_x;
    it.nt = static_cast<int>(q / pix);
    q -= it.nt * pix;
  } else {
    it.nt = static_cast<int>(q % p.n_ntiles);
    q /= p.n_ntiles;
  }
  it.tap0 = 0;
  if (p.up > 1) {
    const int up2 = p.up * p.up;
    it.tap0 = static_cast<int>(q % up2);
    q /= up2;
  }
  it.tx0 = static_cast<int>(q % p.tiles_x) * kTW;
  q /= p.tiles_x;
  it.ty0 = static_cast<int>(q % p.tiles_y) * th;
  it.b = static_cast<int>(q / p.tiles_y);
  return it;
}

template <int N, int MT, bool HALO, int PITCH, bool WS = false>
__global__ void __launch_bounds__(kThreads, 1)
    dense_conv_f16_kernel(const __grid_constant__ CUtensorMap in_map, const Params p) {
  using C = Cfg<N, MT, HALO, PITCH, WS>;
  constexpr int TH = kTH * MT;  // output tile height
  constexpr int H = N / 2;      // accumulator registers of the hi products of one M tile; the cross products follow
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");  // the input image is the previous layer's output
  const int up2 = p.up * p.up;
  const long long n_total = static_cast<long long>(p.B) * p.tiles_y * p.tiles_x * p.n_ntiles * (p.up > 1 ? up2 : 1);
  if (static_cast<long long>(blockIdx.x) >= n_total) return;
  // item sequence of this CTA: round robin (N tile fastest), or for WS a contiguous range (N tile slowest)
  const long long w_first = WS ? (static_cast<long long>(blockIdx.x) * n_total) / gridDim.x : blockIdx.x;
  const long long n_work = WS ? (static_cast<long long>(blockIdx.x + 1) * n_total) / gridDim.x : n_total;
  const long long w_step = WS ? 1 : gridDim.x;
  const long long n_items = (n_work - w_first + w_step - 1) / w_step;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) unsigned long long s_bar[kMaxA + kMaxB + 1];  // activation full[NA] | weight full[NB] | image
  constexpr int kAF = 0, kBF = kMaxA, kWF = kMaxA + kMaxB;

  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127;
  if (tid == 0) {
    for (int s = 0; s < C::NA; ++s) mbar_init(smem_u32(&s_bar[kAF + s]), 1);
    for (int s = 0; s < (WS ? 0 : C::NB); ++s) mbar_init(smem_u32(&s_bar[kBF + s]), 1);
    mbar_init(smem_u32(&s_bar[kWF]), 1);
    fence_mbar_init();
  }
  const uint32_t a_ring = smem_u32(smem);
  const uint32_t b_ring = a_ring + C::NA * C::A_BYTES;
  const int G = p.Cin / 32;
  // steps / activation units per item: HALO: one unit per group, 9 taps each; TAP: one unit per (tap, group)
  const int taps_item = p.up > 1 ? 1 : p.taps;
  const int units_item = HALO ? G : taps_item * G;
  const int steps_item = units_item * C::SPU;
  const long long n_units = n_items * units_item, n_steps = n_items * steps_item;
  auto item_w = [&](long long idx) { return w_first + idx * w_step; };

  // thread 0: activation buffer of global unit a / weight blocks of global step q
  auto issue_a = [&](long long a) {
    const Item im = decode<WS>(item_w(a / units_item), p, TH);
    const int ua = static_cast<int>(a % units_item);
    const int cg0 = p.grouped ? im.nt * G : 0;  // first 32-channel group of this item's input channels
    const uint32_t slot = static_cast<uint32_t>(a % C::NA), bar = smem_u32(&s_bar[kAF + slot]);
    mbar_arrive_expect_tx(bar, static_cast<uint32_t>(C::A_ROWS * 128));
    if (HALO) {
      tma_tile4d(a_ring + slot * C::A_BYTES, &in_map, (cg0 + ua) * 64, im.tx0 - 1, im.ty0 - 1, im.b, bar);
    } else {
      const int t = (p.up > 1 ? im.tap0 : ua / G), g = ua % G;
      const int dy = p.up > 1 ? 0 : t / p.kw, dx = p.up > 1 ? 0 : t % p.kw;
      const int x = im.tx0 * p.stride - p.pad + dx, y = im.ty0 * p.stride - p.pad + dy;  // may be negative: zero fill
      tma_tile4d(a_ring + slot * C::A_BYTES, &in_map, (cg0 + g) * 64, x, y, im.b, bar);
    }
  };
  auto issue_b = [&](long long q) {
    const Item im = decode<WS>(item_w(q / steps_item), p, TH);
    const int u = static_cast<int>(q % steps_item);
    int t, g;
    if (HALO) {
      g = u / 9;
      t = u % 9;
    } else {
      t = p.up > 1 ? im.tap0 : u / G;
      g = u % G;
    }
    const uint8_t *w_tile = p.packed_w + static_cast<size_t>(im.nt) * p.taps * (p.Cin / 16) * C::B_BLK;
    const uint32_t slot = static_cast<uint32_t>(q % C::NB), bar = smem_u32(&s_bar[kBF + slot]);
    mbar_arrive_expect_tx(bar, static_cast<uint32_t>(C::B_BYTES));
    bulk_g2s(b_ring + slot * C::B_BYTES, w_tile + (static_cast<size_t>(t) * (p.Cin / 16) + 2 * g) * C::B_BLK,
             static_cast<uint32_t>(C::B_BYTES), bar);
  };

  bool ovf = false;
  long long next_a = 0, next_b = 0;  // thread 0: next unit / step to load
  int cur_nt = -1;                   // WS: N tile whose weight image is resident
  uint32_t img = 0;                  // WS: images loaded so far
  long long q = 0;                   // global step
  float acc[C::ACC];
  for (long long idx = 0; idx < n_items; ++idx) {
    const Item im = decode<WS>(item_w(idx), p, TH);
#pragma unroll
    for (int i = 0; i < C::ACC; ++i) acc[i] = 0.f;
    for (int ua = 0; ua < units_item; ++ua) {
      for (int t = 0; t < C::SPU; ++t, ++q) {
        __syncthreads();  // the wgmma of step q - 1 have retired in both warpgroups
        if (WS && ua == 0 && t == 0 && im.nt != cur_nt) {
          // first item of a run on this N tile: every step of the previous run has completed, replace the image
          if (tid == 0) {
            const uint32_t bar = smem_u32(&s_bar[kWF]);
            mbar_arrive_expect_tx(bar, static_cast<uint32_t>(p.w_bytes));
            const uint8_t *w_tile = p.packed_w + static_cast<size_t>(im.nt) * p.w_bytes;
            for (int off = 0; off < p.w_bytes; off += 16384) {
              const int bytes = p.w_bytes - off < 16384 ? p.w_bytes - off : 16384;
              bulk_g2s(b_ring + static_cast<uint32_t>(off), w_tile + off, static_cast<uint32_t>(bytes), bar);
            }
          }
          mbar_wait(smem_u32(&s_bar[kWF]), img & 1u);
          ++img;
          cur_nt = im.nt;
        }
        if (tid == 0) {
          for (; next_a < n_units && (next_a - C::NA + 1) * C::SPU <= q; ++next_a) issue_a(next_a);
          if (!WS)
            for (; next_b < n_steps && next_b <= q + C::NB - 1; ++next_b) issue_b(next_b);
        }
        const long long ga = q / C::SPU;  // global unit of this step
        const uint32_t sa = static_cast<uint32_t>(ga % C::NA), sb = static_cast<uint32_t>(q % C::NB);
        mbar_wait(smem_u32(&s_bar[kAF + sa]), static_cast<uint32_t>((ga / C::NA) & 1));
        if (!WS) mbar_wait(smem_u32(&s_bar[kBF + sb]), static_cast<uint32_t>((q / C::NB) & 1));
        const uint32_t a_base = a_ring + sa * C::A_BYTES;
        const uint32_t b_base = WS ? b_ring + static_cast<uint32_t>((t * (p.Cin / 16) + 2 * ua) * C::B_BLK)
                                   : b_ring + sb * C::B_BYTES;
        wg_fence();
#pragma unroll
        for (int kb = 0; kb < 2; ++kb) {
          const uint32_t bk = b_base + static_cast<uint32_t>(kb * C::B_BLK);
          const uint64_t dbh = smem_desc(bk, 2 * N * 16, 128), dbl = smem_desc(bk + N * 16, 2 * N * 16, 128);
#pragma unroll
          for (int mt = 0; mt < MT; ++mt) {
            uint32_t a0, sbo;
            if (HALO) {  // this warpgroup's 8 image rows of M tile mt, shifted by the tap
              a0 = a_base + static_cast<uint32_t>(((mt * kTH + wg * 8 + t / 3) * PITCH + t % 3) * 128);
              sbo = PITCH * 128;
            } else {
              a0 = a_base + static_cast<uint32_t>((mt * kM + wg * 64) * 128);
              sbo = 1024;
            }
            const uint32_t ah = a0 + kb * 32, al = a0 + (2 + kb) * 32;
            const uint32_t bo = p.base_offset_mode ? 1u : 0u;
            const uint64_t dah = gmma_desc(ah, 16, sbo, 1, bo * ((ah >> 7) & 7u)), dal = gmma_desc(al, 16, sbo, 1, bo * ((al >> 7) & 7u));
            float *d = acc + mt * N;
            wg::mma_f16<N>(d, dah, dbh, 1u);      // A_hi x B_hi
            wg::mma_f16<N>(d + H, dah, dbl, 1u);  // A_hi x B_lo'
            wg::mma_f16<N>(d + H, dal, dbh, 1u);  // A_lo' x B_hi
          }
        }
        wg_commit();
        wg_wait<0>();
      }
    }
    wg_fence_acc<C::ACC>(acc);

    // ------------------------------------------------------------------------------------------ epilogue
    const int g_cnt = p.grouped ? __ldg(p.grp_cnt + im.nt) : 0, g_p0 = p.grouped ? __ldg(p.grp_plane0 + im.nt) : 0;
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
      for (int i = 0; i < H; i += 2) {
        const int m = wg * 64 + frag_row(i, wtid), c = frag_col(i, wtid);  // pixel of the M tile, column of the N tile
        const int iy = im.ty0 + mt * kTH + m / kTW, ix = im.tx0 + m % kTW;
        const int ch = im.nt * N + c;  // output channel
        if (iy >= p.oH || ix >= p.oW || (p.grouped ? c >= g_cnt : ch >= p.cout)) continue;
        const int Y = iy * p.up + (p.up > 1 ? im.tap0 / p.up : 0), X = ix * p.up + (p.up > 1 ? im.tap0 % p.up : 0);
        const size_t opix = (static_cast<size_t>(im.b) * p.out_H + Y) * p.out_W + X;
        float v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const bool okc = p.grouped ? true : ch + e < p.cout;
          const float sc = (p.scale && okc) ? __ldg(p.scale + ch + e) : 1.0f, sh = (p.shift && okc) ? __ldg(p.shift + ch + e) : 0.0f;
          float o = fmaf(acc[mt * N + H + i + e], kLoInv, acc[mt * N + i + e]);
          o = fmaf(o, sc, sh);
          if (p.relu) o = fmaxf(o, 0.f);
          v[e] = o;
        }
        if (p.out_h16) {  // channel counts of H16 layers are multiples of 16: whole pairs
          __half h0, l0, h1, l1;
          split_h16(v[0], h0, l0, ovf);
          split_h16(v[1], h1, l1, ovf);
          const int oc = p.out_c0 + ch;
          uint8_t *op = p.out_h16 + opix * (4 * static_cast<size_t>(p.out_C)) + (oc / 32) * 128 + (oc % 32) * 2;
          *reinterpret_cast<__half2 *>(op) = __halves2half2(h0, h1);
          *reinterpret_cast<__half2 *>(op + 64) = __halves2half2(l0, l1);
        }
        if (p.out_nchw) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (p.grouped) {
              if (c + e < g_cnt) p.out_nchw[((static_cast<size_t>(im.b) * p.cout + g_p0 + c + e) * p.out_H + Y) * p.out_W + X] = v[e];
            } else if (ch + e < p.cout) {
              p.out_nchw[((static_cast<size_t>(im.b) * p.cout + ch + e) * p.out_H + Y) * p.out_W + X] = v[e];
            }
          }
        }
      }
    }
  }
  if (ovf && p.status) atomicOr(p.status, 1);
}

// fp32 NCHW image -> pixel H16 rows (32 x 32 tile transpose through shared memory)
__global__ void __launch_bounds__(256) nchw_to_pixel_h16_kernel(const float *__restrict__ in, int C, long long HW,
                                                                __half *__restrict__ out, int32_t *status) {
  __shared__ float s_t[32][33];
  const int b = blockIdx.z;
  const long long p0 = static_cast<long long>(blockIdx.x) * 32;
  const int c0 = blockIdx.y * 32;  // one 32-channel H16 group
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int k = ty; k < 32; k += 8) {
    const int c = c0 + k;
    const long long px = p0 + tx;
    s_t[k][tx] = (c < C && px < HW) ? in[(static_cast<size_t>(b) * C + c) * HW + px] : 0.f;
  }
  __syncthreads();
  bool ovf = false;
  for (int k = ty; k < 32; k += 8) {
    const long long px = p0 + k;
    if (px < HW) {
      __half h, l;
      split_h16(s_t[tx][k], h, l, ovf);
      __half *grp = out + (static_cast<size_t>(b) * HW + px) * (2 * static_cast<size_t>(C)) + static_cast<size_t>(c0) * 2;
      grp[tx] = h;
      grp[32 + tx] = l;
    }
  }
  if (ovf && status) atomicOr(status, 1);
}

// pixel H16 rows -> fp32 NCHW (tests / debugging)
__global__ void __launch_bounds__(256) pixel_h16_to_nchw_kernel(const __half *__restrict__ in, int C, long long HW,
                                                                float *__restrict__ out, long long total) {
  const long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (q >= total) return;
  const long long px = q % HW;
  const int c = static_cast<int>((q / HW) % C);
  const long long b = q / (HW * C);
  const __half *grp = in + (b * HW + px) * (2 * static_cast<long long>(C)) + (c / 32) * 64;
  out[q] = fmaf(__half2float(grp[32 + c % 32]), kLoInv, __half2float(grp[c % 32]));
}

inline int make_image_map(const void *img, int B, int H, int W, int Cin, int stride, int box_x, int box_y, CUtensorMap *map) {
  // Cin = channels per pixel of the image in memory
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
  const cuuint64_t row = static_cast<cuuint64_t>(4) * Cin;  // bytes per pixel
  const cuuint64_t gdim[4] = {static_cast<cuuint64_t>(2 * Cin), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H),
                              static_cast<cuuint64_t>(B)};
  const cuuint64_t gstride[3] = {row, row * W, row * W * H};
  // with an element stride s the box extent is s x the number of elements loaded (cuda.h, cuTensorMapEncodeTiled)
  const cuuint32_t box[4] = {64u, static_cast<cuuint32_t>(box_x * stride), static_cast<cuuint32_t>(box_y * stride), 1u};
  const cuuint32_t estride[4] = {1u, static_cast<cuuint32_t>(stride), static_cast<cuuint32_t>(stride), 1u};
  const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void *>(img), gdim, gstride, box, estride,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? P3D_OK : P3D_ERR_INVALID_ARG;
}

template <int N, int MT, bool HALO, int PITCH, bool WS = false>
int launch(const CUtensorMap &map, const Params &p, cudaStream_t st) {
  using C = Cfg<N, MT, HALO, PITCH, WS>;
  const size_t smem = static_cast<size_t>(C::NA) * C::A_BYTES +
                      (WS ? static_cast<size_t>(p.w_bytes) : static_cast<size_t>(C::NB) * C::B_BYTES) + 1024;
  if (smem > static_cast<size_t>(227 - 6) * 1024) return P3D_ERR_UNSUPPORTED;
  auto kern = dense_conv_f16_kernel<N, MT, HALO, PITCH, WS>;
  P3D_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  const long long work = static_cast<long long>(p.B) * p.tiles_y * p.tiles_x * p.n_ntiles * (p.up > 1 ? p.up * p.up : 1);
  cudaLaunchConfig_t cfg = {};
  const long long sms = num_sms();
  cfg.gridDim = dim3(static_cast<unsigned int>(work < sms ? work : sms));
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  P3D_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, map, p));
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// CenterHead output convs with the 9 taps in the N dimension ("tap-as-N", center_head.py:80-117 SeparateHead finals).
//
// A 3x3 conv with <= 3 output channels is 9 * Cin/16 k-steps of N = 16 MMAs per 128 pixels in the generic kernel above.
// Here one item is a 16 x 16-pixel haloed tile (256 rows = 2 M tiles) of one group's Cin channels and ONE GEMM
//     P[pixel][tap * 3 + co] = sum_c  mid[pixel][c] * W[tap][c][co]            (N = 27 -> 32, K = Cin: 4 k-steps for 64)
// the epilogue parks P in shared memory and every output pixel of the 14 x 14 interior adds its 9 shifted
// entries  out[y][x][co] = bias + sum_tap P[(y + dy) * 16 + x + dx][tap * 3 + co].  The kernel is then bound by reading
// the intermediate image once (x 1.31 halo overhead, mostly L2 hits).
//   step = one 32-channel group of an item (activation ring, NA); the item's weights (all groups) are one slot of a
//   3-deep weight ring; thread 0 loads both ahead across items, warpgroup g computes rows 64g .. 64g+63 of both M tiles.
namespace out9 {
constexpr int kHT = 16, kOT = 14;                 // haloed / output tile side
constexpr int kRows = kHT * kHT;                  // 256 rows of 128 bytes per 32-channel group
constexpr int kABytes = kRows * 128;              // 32 KB
constexpr int kN = 32, kStride = 29;              // GEMM N, fp32 row stride of P in shared memory
constexpr int kWBlk = 64 * kN;                    // bytes of one 16-channel weight k-block ([2 chunks][2N rows][8 halfs])
constexpr int kPBytes = kRows * kStride * 4;
constexpr int kMaxNA = 5, kNW = 3;
constexpr int kAcc = 2 * kN;                      // two M tiles x (hi | cross) x 16 registers

struct Params {
  int B, H, W, G;              // image, 32-channel groups per conv group (Cin / 32)
  int tiles_x, tiles_y, groups, planes, NA;
  const uint8_t *packed_w;     // [groups][Cin / 16] k-blocks of W2[c][tap * 3 + co] (kWBlk bytes each)
  const float *bias;           // [groups][4]
  const int32_t *cin0;         // [groups] first input channel of the group's slice (multiple of 32) or null: g * Cin
  const int32_t *plane0, *cnt; // [groups]
  float *out;                  // [B, planes, H, W]
};

__global__ void __launch_bounds__(kThreads, 1) head_out9_kernel(const __grid_constant__ CUtensorMap in_map, const Params p) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const long long n_work = static_cast<long long>(p.B) * p.tiles_y * p.tiles_x * p.groups;
  if (static_cast<long long>(blockIdx.x) >= n_work) return;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) unsigned long long s_bar[kMaxNA + kNW];
  constexpr int kAF = 0, kWF = kMaxNA;
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127;
  const int NA = p.NA, G = p.G;
  const uint32_t w_slot = static_cast<uint32_t>(2 * G * kWBlk);
  if (tid == 0) {
    for (int s = 0; s < NA; ++s) mbar_init(smem_u32(&s_bar[kAF + s]), 1);
    for (int s = 0; s < kNW; ++s) mbar_init(smem_u32(&s_bar[kWF + s]), 1);
    fence_mbar_init();
  }
  const uint32_t a_ring = smem_u32(smem);
  const uint32_t w_ring = a_ring + static_cast<uint32_t>(NA * kABytes);
  float *s_p = reinterpret_cast<float *>(smem + static_cast<size_t>(NA) * kABytes + static_cast<size_t>(kNW) * w_slot);

  auto decode = [&](long long w, int &g, int &tx0, int &ty0, int &b) {
    g = static_cast<int>(w % p.groups);
    long long q = w / p.groups;
    tx0 = static_cast<int>(q % p.tiles_x) * kOT;
    q /= p.tiles_x;
    ty0 = static_cast<int>(q % p.tiles_y) * kOT;
    b = static_cast<int>(q / p.tiles_y);
  };
  const long long n_items = (n_work - blockIdx.x + gridDim.x - 1) / gridDim.x;
  const long long n_steps = n_items * G;
  // thread 0: activation tile of global step q (item q / G, group q % G) / weights of item i
  auto issue_a = [&](long long q) {
    int g, tx0, ty0, b;
    decode(blockIdx.x + (q / G) * gridDim.x, g, tx0, ty0, b);
    const int cg0 = (p.cin0 ? __ldg(p.cin0 + g) : g * G * 32) / 32;
    const uint32_t slot = static_cast<uint32_t>(q % NA), bar = smem_u32(&s_bar[kAF + slot]);
    mbar_arrive_expect_tx(bar, static_cast<uint32_t>(kABytes));
    tma_tile4d(a_ring + slot * kABytes, &in_map, (cg0 + static_cast<int>(q % G)) * 64, tx0 - 1, ty0 - 1, b, bar);
  };
  auto issue_w = [&](long long i) {
    const int g = static_cast<int>((blockIdx.x + i * gridDim.x) % p.groups);
    const uint32_t slot = static_cast<uint32_t>(i % kNW), bar = smem_u32(&s_bar[kWF + slot]);
    mbar_arrive_expect_tx(bar, w_slot);
    bulk_g2s(w_ring + slot * w_slot, p.packed_w + static_cast<size_t>(g) * w_slot, w_slot, bar);
  };

  long long next_a = 0, next_w = 0, q = 0;
  float acc[kAcc];
  for (long long idx = 0; idx < n_items; ++idx) {
    int g, tx0, ty0, b;
    decode(blockIdx.x + idx * gridDim.x, g, tx0, ty0, b);
    const int cnt = __ldg(p.cnt + g), p0 = __ldg(p.plane0 + g);
    const float4 bias = __ldg(reinterpret_cast<const float4 *>(p.bias) + g);
#pragma unroll
    for (int i = 0; i < kAcc; ++i) acc[i] = 0.f;
    const uint32_t ws = static_cast<uint32_t>(idx % kNW);
    for (int k = 0; k < G; ++k, ++q) {
      __syncthreads();  // the wgmma of step q - 1 have retired in both warpgroups
      if (tid == 0) {
        for (; next_a < n_steps && next_a <= q + NA - 1; ++next_a) issue_a(next_a);
        for (; next_w < n_items && (next_w - kNW + 1) * G <= q; ++next_w) issue_w(next_w);
      }
      if (k == 0) mbar_wait(smem_u32(&s_bar[kWF + ws]), static_cast<uint32_t>((idx / kNW) & 1));
      const uint32_t sa = static_cast<uint32_t>(q % NA);
      mbar_wait(smem_u32(&s_bar[kAF + sa]), static_cast<uint32_t>((q / NA) & 1));
      const uint32_t a_base = a_ring + sa * kABytes;
      const uint32_t w_base = w_ring + ws * w_slot;
      wg_fence();
#pragma unroll
      for (int kb = 0; kb < 2; ++kb) {
        const uint32_t bk = w_base + static_cast<uint32_t>((k * 2 + kb) * kWBlk);
        const uint64_t dbh = smem_desc(bk, 2 * kN * 16, 128), dbl = smem_desc(bk + kN * 16, 2 * kN * 16, 128);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          const uint32_t a0 = a_base + static_cast<uint32_t>((mt * kM + wg * 64) * 128);
          const uint64_t dah = desc_sw128(a0 + kb * 32), dal = desc_sw128(a0 + (2 + kb) * 32);
          float *d = acc + mt * kN;
          wg::mma_f16<kN>(d, dah, dbh, 1u);
          wg::mma_f16<kN>(d + kN / 2, dah, dbl, 1u);
          wg::mma_f16<kN>(d + kN / 2, dal, dbh, 1u);
        }
      }
      wg_commit();
      wg_wait<0>();
    }
    wg_fence_acc<kAcc>(acc);
    // P[row][col] = hi + cross * 2^-11 for the 27 used columns
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
      for (int i = 0; i < kN / 2; ++i) {
        const int r = mt * kM + wg * 64 + frag_row(i, wtid), c = frag_col(i, wtid);
        if (c < 27) s_p[r * kStride + c] = fmaf(acc[mt * kN + kN / 2 + i], kLoInv, acc[mt * kN + i]);
      }
    }
    __syncthreads();
    for (int o = tid; o < kOT * kOT; o += kThreads) {
      const int oy = o / kOT, ox = o - oy * kOT;
      const int Y = ty0 + oy, X = tx0 + ox;
      if (Y < p.H && X < p.W) {
        float s0 = bias.x, s1 = bias.y, s2 = bias.z;
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          const float *e = s_p + ((oy + t / 3) * kHT + ox + t % 3) * kStride + t * 3;
          s0 += e[0];
          s1 += e[1];
          s2 += e[2];
        }
        float *op = p.out + ((static_cast<size_t>(b) * p.planes + p0) * p.H + Y) * p.W + X;
        const size_t plane = static_cast<size_t>(p.H) * p.W;
        op[0] = s0;
        if (cnt > 1) op[plane] = s1;
        if (cnt > 2) op[2 * plane] = s2;
      }
    }
  }
}
}  // namespace out9

}  // namespace dcf
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_nchw_to_pixel_h16(const float *in, int B, int C, int H, int W, void *out_h16, int32_t *status_dev,
                                     p3d_stream_t stream) {
  if (!in || !out_h16 || B < 1 || C < 32 || C % 32 || H < 1 || W < 1) return P3D_ERR_INVALID_ARG;
  const long long hw = static_cast<long long>(H) * W;
  dim3 grid(static_cast<unsigned int>((hw + 31) / 32), static_cast<unsigned int>(C / 32), B);
  dcf::nchw_to_pixel_h16_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(in, C, hw, static_cast<__half *>(out_h16),
                                                                                      status_dev);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" int p3d_pixel_h16_to_nchw(const void *in_h16, int B, int C, int H, int W, float *out, p3d_stream_t stream) {
  if (!in_h16 || !out || B < 1 || C < 32 || C % 32 || H < 1 || W < 1) return P3D_ERR_INVALID_ARG;
  const long long hw = static_cast<long long>(H) * W, total = hw * C * B;
  dcf::pixel_h16_to_nchw_kernel<<<div_up(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half *>(in_h16), C, hw, out, total);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

// packed weights: per N tile the image p3d_sparse_conv_f16_pack_weights makes of W[tap][Cin][n_tile] (zero-padded columns)
extern "C" size_t p3d_dense_conv2d_f16_packed_weight_bytes(int taps, int Cin, int Cout, int n_tile) {
  if (taps < 1 || Cin < 32 || Cin % 32 || Cout < 1 || (n_tile != 16 && n_tile != 32 && n_tile != 64 && n_tile != 128)) return 0;
  const size_t tiles = static_cast<size_t>((Cout + n_tile - 1) / n_tile);
  return align_up(tiles * taps * Cin * static_cast<size_t>(n_tile) * 4);
}

// mode: 0 auto (HALO for 3x3 stride 1 pad 1 convolutions - weight-stationary when it applies -, TAP otherwise), 1 force TAP,
// 2 force the weight-stationary kernel (P3D_ERR_UNSUPPORTED when it does not apply); m_tiles: 0 auto, 1 or 2
static int dense_conv_f16(const void *in_h16, int B, int H, int W, int Cin, const void *packed_weight, int Cout, int n_tile,
                          int kh, int kw, int stride, int pad, int up, const float *scale, const float *shift, int relu,
                          void *out_h16, int out_C, int out_c0, float *out_nchw, int mode, int m_tiles, int32_t *status_dev,
                          p3d_stream_t stream, int groups, int in_C, const int32_t *grp_plane0, const int32_t *grp_cnt) {
  if (!in_h16 || !packed_weight || (!out_h16 && !out_nchw) || B < 1 || H < 1 || W < 1 || Cout < 1) return P3D_ERR_INVALID_ARG;
  if (Cin < 32 || Cin % 32 || (n_tile != 64 && n_tile != 128 && !(groups && n_tile == 16))) return P3D_ERR_UNSUPPORTED;
  if (up < 1 || (up > 1 && (kh != up || kw != up || stride != up || pad != 0))) return P3D_ERR_UNSUPPORTED;
  if (up == 1 && (kh < 1 || kw < 1 || kh * kw > 32 || stride < 1 || stride > 2 || pad < 0)) return P3D_ERR_UNSUPPORTED;
  if (out_h16 && (Cout % 16 || out_C % 32 || out_c0 % 16 || out_c0 + Cout > out_C)) return P3D_ERR_INVALID_ARG;
  if ((reinterpret_cast<uintptr_t>(in_h16) & 15) || (reinterpret_cast<uintptr_t>(packed_weight) & 15) ||
      (reinterpret_cast<uintptr_t>(out_h16) & 15))
    return P3D_ERR_INVALID_ARG;
  dcf::Params p;
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
  p.n_ntiles = groups ? groups : (Cout + n_tile - 1) / n_tile;
  p.cout = Cout;
  p.grouped = groups ? 1 : 0;
  p.in_C = groups ? in_C : Cin;
  p.grp_plane0 = grp_plane0;
  p.grp_cnt = grp_cnt;
  p.out_C = out_C;
  p.out_c0 = out_c0;
  p.relu = relu;
  p.packed_w = static_cast<const uint8_t *>(packed_weight);
  p.scale = scale;
  p.shift = shift;
  p.out_h16 = static_cast<uint8_t *>(out_h16);
  p.out_nchw = out_nchw;
  p.status = status_dev;
  static const int env_mode = getenv("P3D_DENSE_MODE") ? atoi(getenv("P3D_DENSE_MODE")) : -1;  // tuning hooks
  static const int env_mt = getenv("P3D_DENSE_MT") ? atoi(getenv("P3D_DENSE_MT")) : -1;
  static const int env_pitch = getenv("P3D_DENSE_PITCH") ? atoi(getenv("P3D_DENSE_PITCH")) : 10;
  // shifted tiles read correctly with base_offset = 0: the swizzle is a function of the absolute shared-memory address
  // (tests/test_gpu_dense.py); P3D_DENSE_BO=1 sets it to the address bits 7-9 instead
  static const int env_bo = getenv("P3D_DENSE_BO") ? atoi(getenv("P3D_DENSE_BO")) : 0;
  p.base_offset_mode = env_bo;
  const int pitch = env_pitch == 16 ? 16 : 10;
  if (env_mode >= 0) mode = env_mode;
  if (env_mt >= 0) m_tiles = env_mt;
  const bool halo = (mode == 0 || mode == 2) && up == 1 && kh == 3 && kw == 3 && stride == 1 && pad == 1;
  // two M tiles per item (half the weight traffic per flop) when that still leaves every SM an item
  int mt = m_tiles;
  if (mt != 1 && mt != 2) {
    const long long tx = (p.oW + dcf::kTW - 1) / dcf::kTW, ty2 = (p.oH + 2 * dcf::kTH - 1) / (2 * dcf::kTH);
    const long long items2 = static_cast<long long>(B) * tx * ty2 * p.n_ntiles * (up > 1 ? up * up : 1);
    // two M tiles for the narrow N = 64 layers (the second tile halves the weight traffic per flop and amortises the
    // per-item prologue) when that still leaves every SM an item; N = 128 keeps one (register budget)
    mt = (n_tile <= 64 && items2 >= (num_sms() * 9) / 10) ? 2 : 1;
  }
  // weight-stationary variant: haloed 3x3, N tile 64, the N tile's weight image + 3 activation tiles fit in shared memory,
  // and every CTA has enough pixel tiles per weight image to amortise loading it (mode 2 forces it, P3D_DENSE_WS=0 disables)
  // The variant is OFF unless asked for (mode 2 or P3D_DENSE_WS=1): it was not faster than the streaming N = 128 kernel on
  // the CenterHead's 64 -> 2304 layer.
  static const int env_ws = getenv("P3D_DENSE_WS") ? atoi(getenv("P3D_DENSE_WS")) : 0;
  p.w_bytes = p.taps * (Cin / 16) * 64 * n_tile;
  bool ws = false;
  if (halo && n_tile == 64 && !groups && pitch == 10 && (env_ws || mode == 2)) {
    const size_t need = 3 * static_cast<size_t>(dcf::Cfg<64, 1, true, 10, true>::A_BYTES) + p.w_bytes + 1024;
    const long long pix = static_cast<long long>(B) * ((p.oW + dcf::kTW - 1) / dcf::kTW) * ((p.oH + dcf::kTH - 1) / dcf::kTH);
    const long long items = pix * p.n_ntiles;
    ws = need <= static_cast<size_t>(227 - 6) * 1024 && (mode == 2 || items >= 8ll * num_sms());
  }
  if (mode == 2 && !ws) return P3D_ERR_UNSUPPORTED;
  if (ws || n_tile > 64) mt = 1;  // two M tiles of a 128-wide N tile would need 256 accumulator registers per thread
  p.tiles_x = (p.oW + dcf::kTW - 1) / dcf::kTW;
  p.tiles_y = (p.oH + dcf::kTH * mt - 1) / (dcf::kTH * mt);
  CUtensorMap map;
  const int bx = halo ? pitch : dcf::kTW, by = halo ? dcf::kTH * mt + 2 : dcf::kTH * mt;
  const int rc = dcf::make_image_map(in_h16, B, H, W, p.in_C, p.stride, bx, by, &map);
  if (rc != P3D_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (ws) return dcf::launch<64, 1, true, 10, true>(map, p, st);
#define P3D_DCF(NT, M)                                                                          \
  if (n_tile == NT && mt == M) {                                                                \
    if (!halo) return dcf::launch<NT, M, false, 10>(map, p, st);                                \
    if (pitch == 16) return dcf::launch<NT, M, true, 16>(map, p, st);                           \
    return dcf::launch<NT, M, true, 10>(map, p, st);                                            \
  }
  P3D_DCF(16, 1)
  P3D_DCF(16, 2)
  P3D_DCF(64, 1)
  P3D_DCF(64, 2)
  P3D_DCF(128, 1)
#undef P3D_DCF
  return P3D_ERR_UNSUPPORTED;
}

extern "C" int p3d_dense_conv2d_f16(const void *in_h16, int B, int H, int W, int Cin, const void *packed_weight, int Cout,
                                    int n_tile, int kh, int kw, int stride, int pad, int up, const float *scale,
                                    const float *shift, int relu, void *out_h16, int out_C, int out_c0, float *out_nchw,
                                    int mode, int m_tiles, int32_t *status_dev, p3d_stream_t stream) {
  return dense_conv_f16(in_h16, B, H, W, Cin, packed_weight, Cout, n_tile, kh, kw, stride, pad, up, scale, shift, relu, out_h16,
                        out_C, out_c0, out_nchw, mode, m_tiles, status_dev, stream, 0, 0, nullptr, nullptr);
}

// Grouped 3x3 / stride 1 / pad 1 output convs (CenterHead SeparateHead finals, center_head.py:80-117) on the tensor cores:
// group g convolves input channels [g * Cin, (g + 1) * Cin) of the in_C-channel image with its own W[9][Cin][16]
// (columns >= cnt[g] zero) and writes cnt[g] fp32 planes from plane0[g] of out_nchw [B, planes, H, W].
// packed_weight: `groups` weight tiles of p3d_dense_conv2d_f16_pack_weights(taps 9, Cin, n_tile 16); bias [groups][16].
extern "C" int p3d_grouped_head_conv_f16(const void *in_h16, int B, int H, int W, int in_C, int Cin, int groups,
                                         const void *packed_weight, const float *bias, const int32_t *plane0_dev,
                                         const int32_t *cnt_dev, int planes, float *out_nchw, int32_t *status_dev,
                                         p3d_stream_t stream) {
  if (!plane0_dev || !cnt_dev || groups < 1 || groups * Cin > in_C || in_C % 32 || planes < 1) return P3D_ERR_INVALID_ARG;
  return dense_conv_f16(in_h16, B, H, W, Cin, packed_weight, planes, 16, 3, 3, 1, 1, 1, nullptr, bias, 0, nullptr, 32, 0, out_nchw,
                        0, 0, status_dev, stream, groups, in_C, plane0_dev, cnt_dev);
}

// Output convs of the CenterHead, 9 taps in the GEMM's N dimension (dcf::out9 above): group g convolves input channels
// [cin0[g], cin0[g] + Cin) (cin0 null: g * Cin) of the in_C-channel pixel fp16-pair image with its own 3x3 weights and
// writes cnt[g] <= 3 fp32 planes from plane0[g] of out_nchw [B, planes, H, W].  packed_weight: per group the image
// p3d_dense_conv2d_f16_pack_weights(taps 1, Cin, n_tile 32) makes of W2[c][tap * 3 + co]; bias [groups][4].
extern "C" int p3d_head_out_conv_f16(const void *in_h16, int B, int H, int W, int in_C, int Cin, int groups,
                                     const void *packed_weight, const float *bias, const int32_t *cin0_dev,
                                     const int32_t *plane0_dev, const int32_t *cnt_dev, int planes, float *out_nchw,
                                     p3d_stream_t stream) {
  if (!in_h16 || !packed_weight || !bias || !plane0_dev || !cnt_dev || !out_nchw || B < 1 || H < 1 || W < 1 || groups < 1 ||
      planes < 1 || in_C % 32 || Cin > in_C)
    return P3D_ERR_INVALID_ARG;
  if (Cin != 32 && Cin != 64 && Cin != 128) return P3D_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(in_h16) & 15) || (reinterpret_cast<uintptr_t>(packed_weight) & 15) ||
      (reinterpret_cast<uintptr_t>(bias) & 15))
    return P3D_ERR_INVALID_ARG;
  namespace o9 = dcf::out9;
  o9::Params p;
  p.B = B;
  p.H = H;
  p.W = W;
  p.G = Cin / 32;
  p.tiles_x = (W + o9::kOT - 1) / o9::kOT;
  p.tiles_y = (H + o9::kOT - 1) / o9::kOT;
  p.groups = groups;
  p.planes = planes;
  p.NA = p.G <= 2 ? 5 : 4;
  p.packed_w = static_cast<const uint8_t *>(packed_weight);
  p.bias = bias;
  p.cin0 = cin0_dev;
  p.plane0 = plane0_dev;
  p.cnt = cnt_dev;
  p.out = out_nchw;
  CUtensorMap map;
  const int rc = dcf::make_image_map(in_h16, B, H, W, in_C, 1, o9::kHT, o9::kHT, &map);
  if (rc != P3D_OK) return rc;
  const size_t smem = static_cast<size_t>(p.NA) * o9::kABytes + static_cast<size_t>(o9::kNW) * 2 * p.G * o9::kWBlk + o9::kPBytes + 1024;
  auto kern = o9::head_out9_kernel;
  P3D_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  const long long work = static_cast<long long>(B) * p.tiles_y * p.tiles_x * groups;
  cudaLaunchConfig_t cfg = {};
  const long long sms = num_sms();
  cfg.gridDim = dim3(static_cast<unsigned int>(work < sms ? work : sms));
  cfg.blockDim = dim3(tc::kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  P3D_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, map, p));
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
