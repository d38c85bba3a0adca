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
//   step        (A unit, tap): HALO one A unit per 32-channel group serves 9 steps, TAP one A unit per step.
//   warp-specialized CTA of three warpgroups: warpgroup 0 is the producer - one thread keeps an activation ring (NA) and
//               a weight ring (NB) filled ahead of the consumers across work items (TMA / cp.async.bulk onto "full"
//               mbarriers, refilling a slot once its "empty" mbarrier says both consumers are done with it); consumer
//               warpgroup c = 1, 2 computes rows 64(c-1) .. 64(c-1)+63 of every M tile with one wgmma group in flight
//               behind the one being issued.  At the end of an item it hands its rows to warps 1-3 of warpgroup 0 (the
//               epilogue warps) through its staging tile and starts the next item, so the tensor pipe does not idle
//               through the stores.  A launch that writes only the pixel H16 image stages finished fp16-pair rows
//               (scale / shift / ReLU and the split done by the consumers) that one epilogue thread stores with TMA;
//               a launch with fp32 planes stages hi + cross * 2^-11 in fp32 and the epilogue warps do the rest.
#include <cuda.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "h16.cuh"
#include "p3d_b200.h"
#include "tc_common.cuh"

namespace p3d {
namespace dcf {

using namespace tc;

constexpr int kTW = 8, kTH = 16;        // output tile of one M = 128 tile: 8 x 16 pixels
constexpr int kPitch = kTW + 2;         // pixels per row of the haloed tile in shared memory
constexpr int kMaxA = 6, kMaxB = 12;    // activation / weight ring depth limits
constexpr int kSmemBudget = (227 - 6) * 1024;  // 227 KB per CTA less alignment slack and the static barriers
constexpr int kDenseThreads = 384;      // producer warpgroup + two consumer warpgroups
constexpr uint32_t kConsumerWarps = 8;  // arrivals that release a slot: one per consumer warp
constexpr uint32_t kEpiThreads = 96;    // warps 1-3 of the producer warpgroup: the epilogue warps
constexpr int kFlush = 9;               // steps (18 k-steps) per hi x hi partial before it joins the fp32 total
constexpr int kFlushTerms = 8192;       // products per output above which a launch flushes (FLUSH instantiations)

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
};
// Parameters of the FUSE_P kernel (a separate type keeps the other instantiations' parameter block as it is): per N tile
// the two 64-channel heads' tap-as-N weight images (out9 layout, 2 x kP2Bytes)
struct ParamsP : Params {
  const uint8_t *packed_w2;
};
// Parameters of residual launches (RES): the pixel H16 image [B, out_H, out_W, res_C] whose channels [0, cout) are added
// after scale / shift and before ReLU
struct ParamsR : Params {
  const uint8_t *res_h16;
  int res_C;
};
template <bool FUSE_P, bool RES = false>
using KParams = std::conditional_t<FUSE_P, ParamsP, std::conditional_t<RES, ParamsR, Params>>;

// FUSE_P: the tap-as-N GEMM of the output convs (out9 below) on a staged pair tile.  A 64-channel head's W2 image is
// p3d_dense_conv2d_f16_pack_weights(taps 1, Cin 64, n_tile 32): 4 k-blocks of 2 KB; P rows have kPPitch fp32 columns
// (the 27 used ones and a zero column that keeps a pixel's row 16-byte aligned).
constexpr int kP2Blk = 64 * 32, kP2Bytes = 4 * kP2Blk, kPPitch = 28;

template <int N, int MT, bool HALO>
struct Cfg {
  static constexpr int A_ROWS = HALO ? kPitch * (kTH * MT + 2) : kM * MT;    // rows of 128 bytes per activation buffer
  static constexpr int A_BYTES = ((A_ROWS * 128 + 1023) / 1024) * 1024;
  static constexpr int B_BYTES = 128 * N;                                    // weight blocks of one (tap, group): 2 k-blocks
  static constexpr int B_BLK = 64 * N;
  // Staged epilogue: a consumer warpgroup parks hi + cross * 2^-11 of its rows (MT x 64 rows x N columns, fp32) in its
  // own staging tile and goes on with the next item; the epilogue warps apply scale / shift / ReLU, split and store.
  // Row pitch N + 8 floats: the 32 bytes of padding put the four rows of a half-warp's fragment stores on distinct banks.
  static constexpr int SP = N + 8;                                           // staging row pitch (floats)
  static constexpr int STG_WG = MT * 64 * SP;                                // floats per consumer warpgroup
  static constexpr int STG_BYTES = 2 * STG_WG * 4;
  // Without fp32 planes the same tile holds the fp16-pair rows instead: one 8 KB TMA block per (M tile, 32-channel group)
  // and after them two buffers of the item's N scale and N shift values
  static constexpr int PAIR_BLK = 64 * 128, PAIR_BYTES = MT * (N / 32) * PAIR_BLK;
  static_assert(PAIR_BYTES + 2 * 2 * N * 4 <= STG_WG * 4 && STG_WG * 4 % 1024 == 0, "pair tile inside the staging tile");
  static constexpr int AVAIL = kSmemBudget - STG_BYTES;
  // TAP mode: every step needs a new activation buffer, so both rings get the same depth; HALO: 2 buffers
  static constexpr int NA_TAP_RAW = AVAIL / (A_BYTES + B_BYTES);
  static constexpr int NA = HALO ? 2 : (NA_TAP_RAW > kMaxA ? kMaxA : NA_TAP_RAW);
  static constexpr int BUDGET = AVAIL - NA * A_BYTES;
  static constexpr int NB_RAW = BUDGET / B_BYTES;
  static constexpr int NB = NB_RAW > kMaxB ? kMaxB : NB_RAW;                 // weight ring depth
  static constexpr int ACC = MT * N;                                         // fp32 registers per thread
  static constexpr int SPU = HALO ? 9 : 1;                                   // steps per activation buffer
  // register split, 128 P + 256 C <= 384 x 168 (what a CTA of 384 threads holds at launch); the consumers hold up to 128
  // fp32 accumulators, the producer warpgroup's warps 1-3 run the epilogue.
  static constexpr int P_REGS = 88, C_REGS = 208;
  static_assert(128 * P_REGS + 256 * C_REGS <= kDenseThreads * 168, "register split");
  static_assert(N == 64 || N == 128, "N tile: 64 or 128");
  static_assert(MT == 1 || MT == 2, "one or two M tiles");
  static_assert(MT * N <= 128, "accumulators: at most 128 registers per thread");
  static_assert(NB >= 3, "weight ring too shallow");
  static_assert(NA >= 2 && NA <= kMaxA, "activation ring depth");
};

__device__ __forceinline__ void tma_tile4d(uint32_t dst, const CUtensorMap *map, int c, int x, int y, int b, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];" ::
          "r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c), "r"(x), "r"(y), "r"(b), "r"(bar)
      : "memory");
}
// TMA tensor stores shared -> global into the issuing thread's bulk async-group
__device__ __forceinline__ void tma_store4d(const CUtensorMap *map, uint32_t src, int c, int x, int y, int b) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(src), "r"(c), "r"(x), "r"(y), "r"(b)
               : "memory");
}
__device__ __forceinline__ void tma_store5d(const CUtensorMap *map, uint32_t src, int c, int d1, int d2, int d3, int d4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(src), "r"(c), "r"(d1), "r"(d2), "r"(d3), "r"(d4)
               : "memory");
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v));
}
__device__ __forceinline__ float2 ld_shared_f2(uint32_t addr) {
  float2 v;
  asm("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));  // ordered by its address only
  return v;
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// .read: the shared-memory sources of the committed stores may be overwritten; without: the writes are done
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
struct Item {
  int nt, tap0, tx0, ty0, b;
};

// Trace build (-DP3D_DENSE_TRACE, tools/dense_bench.py --trace): each role sums clock64 intervals of where it waits and
// adds them per CTA to g_dense_trace, which p3d_dense_trace_read copies out.  Without the macro every Trace member is
// empty and the kernel compiles to the code it has without the calls.
enum TraceField {
  kTrItems, kTrCycles,                  // items of the CTA; cycles of consumer warpgroup 1 from start-up to its exit
  kTrAFull, kTrBFull = kTrAFull + 2,    // per consumer warpgroup: waiting on activation / weight "full"
  kTrMma = kTrBFull + 2,                // per consumer warpgroup: in wgmma.wait_group
  kTrEpi = kTrMma + 2,                  // per consumer warpgroup: after the item's last wait_group until the next item
                                        // (writing the staging tile), less kTrStageFree
  kTrStageFree = kTrEpi + 2,            // per consumer warpgroup: waiting for the epilogue warps to free its staging tile
  kTrAEmpty = kTrStageFree + 2, kTrBEmpty,  // producer: waiting on activation / weight "empty"
  kTrEwWait, kTrEwBusy,                 // epilogue thread 0: waiting on "staged"; from "staged" to "freed" (fp32
                                        // staging: scale / shift / ReLU / split and stores; pair tile: the TMA stores
                                        // until their shared-memory reads are done)
  kTrFields
};
#ifdef P3D_DENSE_TRACE
constexpr int kTrMaxCtas = 1024;
__device__ unsigned long long g_dense_trace[kTrMaxCtas][kTrFields];
struct Trace {
  unsigned long long sum[kTrFields] = {};
  __device__ __forceinline__ long long now() const { return clock64(); }
  __device__ __forceinline__ void add(int f, long long t0) { sum[f] += static_cast<unsigned long long>(clock64() - t0); }
  __device__ __forceinline__ void count(int f, unsigned long long v) { sum[f] += v; }
  // per-warpgroup fields are summed in the first of their pair and land in pair entry cw
  __device__ void flush(int cw) const {
#pragma unroll
    for (int f = 0; f < kTrFields; ++f) {
      const int dst = f >= kTrAFull && f < kTrAEmpty ? f + cw : f;
      if (sum[f]) atomicAdd(&g_dense_trace[blockIdx.x % kTrMaxCtas][dst], sum[f]);
    }
  }
};
#else
struct Trace {
  __device__ __forceinline__ long long now() const { return 0; }
  __device__ __forceinline__ void add(int, long long) {}
  __device__ __forceinline__ void count(int, unsigned long long) {}
  __device__ __forceinline__ void flush(int) const {}
};
#endif
// item idx of this CTA: round robin over the grid, N tile fastest
__device__ __forceinline__ Item decode(long long idx, const Params &p, int th) {
  Item it;
  long long q = blockIdx.x + idx * gridDim.x;
  it.nt = static_cast<int>(q % p.n_ntiles);
  q /= p.n_ntiles;
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

// Epilogue warps (warps 1-3 of the producer warpgroup, thread et = 0 .. 95).  For every item, and for consumer warpgroup
// c = 0, 1 in turn: wait until c has staged its rows, apply scale / shift and ReLU, write the outputs, and hand the tile
// back.  Pixel H16 rows: a lane takes four channels of one pixel, so eight lanes write one pixel's 32-channel group as 64
// contiguous bytes of hi and 64 of lo'.  fp32 NCHW planes: a lane takes one pixel of an 8-pixel tile row, so eight lanes
// write 32 contiguous bytes of a plane.
template <int N, int MT>
__device__ __forceinline__ void epilogue_warps(const Params &p, const float *stg, unsigned long long *staged,
                                               unsigned long long *freed, long long n_items, int th, int et) {
  constexpr int SP = N + 8, ROWS = MT * 64;  // staging row pitch (floats) and rows per consumer warpgroup (Cfg)
  const int ew = et >> 5, lane = et & 31;
  bool ovf = false;
  Trace tr;
  for (long long idx = 0; idx < n_items; ++idx) {
    const Item im = decode(idx, p, th);
    const int dy = p.up > 1 ? im.tap0 / p.up : 0, dx = p.up > 1 ? im.tap0 % p.up : 0;
    for (int c = 0; c < 2; ++c) {
      long long t0 = tr.now();
      mbar_wait(smem_u32(staged + c), static_cast<uint32_t>(idx & 1));
      tr.add(kTrEwWait, t0);
      t0 = tr.now();
      const float *st = stg + c * ROWS * SP;
      // staging row r of consumer c is pixel c * 64 + r % 64 of M tile r / 64; false outside the output
      auto pixel = [&](int r, int &Y, int &X) {
        const int m = c * 64 + (r & 63), iy = im.ty0 + (r >> 6) * kTH + m / kTW, ix = im.tx0 + m % kTW;
        Y = iy * p.up + dy;
        X = ix * p.up + dx;
        return iy < p.oH && ix < p.oW;
      };
      if (p.out_h16) {
        const int r4 = lane >> 3, c4 = (lane & 7) * 4;  // row of a 4-row quad, first of four columns
        for (int q = 0; q < N / 32; ++q) {
          const int col = q * 32 + c4, ch = im.nt * N + col, oc = p.out_c0 + ch;
          // channel counts of H16 layers are multiples of 16: the four columns are valid together
          if (ch >= p.cout) continue;
          float sc[4], sh[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            sc[e] = p.scale ? __ldg(p.scale + ch + e) : 1.0f;
            sh[e] = p.shift ? __ldg(p.shift + ch + e) : 0.0f;
          }
#pragma unroll 2
          for (int rq = ew; rq < ROWS / 4; rq += 3) {
            const int r = rq * 4 + r4;
            int Y, X;
            if (!pixel(r, Y, X)) continue;
            const float4 o4 = *reinterpret_cast<const float4 *>(st + r * SP + col);
            float v[4] = {o4.x, o4.y, o4.z, o4.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              v[e] = fmaf(v[e], sc[e], sh[e]);
              if (p.relu) v[e] = fmaxf(v[e], 0.f);
            }
            __half2 h01, l01, h23, l23;
            split_h16x2(v[0], v[1], h01, l01, ovf);
            split_h16x2(v[2], v[3], h23, l23, ovf);
            uint8_t *op = p.out_h16 + ((static_cast<size_t>(im.b) * p.out_H + Y) * p.out_W + X) * (4 * static_cast<size_t>(p.out_C)) +
                          (oc / 32) * 128 + (oc % 32) * 2;
            *reinterpret_cast<uint2 *>(op) = make_uint2(*reinterpret_cast<const uint32_t *>(&h01), *reinterpret_cast<const uint32_t *>(&h23));
            *reinterpret_cast<uint2 *>(op + 64) = make_uint2(*reinterpret_cast<const uint32_t *>(&l01), *reinterpret_cast<const uint32_t *>(&l23));
          }
        }
      }
      if (p.out_nchw) {
        const int px = lane & 7, cc = lane >> 3;  // pixel of an 8-pixel tile row, channel of a 4-channel quad
        for (int u = ew; u < (ROWS / 8) * (N / 4); u += 3) {
          const int r = (u % (ROWS / 8)) * 8 + px, col = (u / (ROWS / 8)) * 4 + cc, ch = im.nt * N + col;
          int Y, X;
          if (ch >= p.cout || !pixel(r, Y, X)) continue;
          const float sc = p.scale ? __ldg(p.scale + ch) : 1.0f, sh = p.shift ? __ldg(p.shift + ch) : 0.0f;
          float v = fmaf(st[r * SP + col], sc, sh);
          if (p.relu) v = fmaxf(v, 0.f);
          p.out_nchw[((static_cast<size_t>(im.b) * p.cout + ch) * p.out_H + Y) * p.out_W + X] = v;
        }
      }
      mbar_arrive(smem_u32(freed + c));
      tr.add(kTrEwBusy, t0);
    }
  }
  if (ovf && p.status) atomicOr(p.status, 1);
  if (et == 0) tr.flush(0);
}

// Pair-tile epilogue (launches without fp32 planes).  The consumers have applied scale / shift / ReLU and the split and
// staged fp16-pair rows in the layout a SWIZZLE_128B TMA box lands in: one 8 KB block per (M tile, 32-channel group) of
// 64 rows x 128 bytes, row = pixel y * 8 + x of the warpgroup's 8 x 8 pixels, 16-byte chunk XOR-ed with row & 7.  Thread
// et = 0 stores every block whose 32 channels the layer owns with TMA (a transposed conv: one box per input-pixel row,
// rows below the image skipped so that a ragged tile does not spill into the next batch image) and hands the tile back
// once the stores have read it.  A box over a group the layer owns in part (out_c0 % 32 == 16, or the last group of a
// partly used N tile) would overwrite the neighbour's channels: all 96 threads copy the owned 32-byte hi and lo' halves
// of such blocks with ordinary stores.  FUSE_P: the consumers have staged the item's two P groups instead ([group][64
// rows][kPPitch] fp32), which thread 0 stores as one box of the P buffer (make_p_map).
template <int N, int MT, bool FUSE_P>
__device__ __forceinline__ void epilogue_pairs(const Params &p, const CUtensorMap *out_map, const uint8_t *tiles, int tile_bytes,
                                               unsigned long long *staged, unsigned long long *freed, long long n_items,
                                               int th, int et) {
  constexpr int NQ = N / 32, BLK = 64 * 128;
  const bool lead = et == 0;
  const bool whole = p.out_c0 % 32 == 0;  // output groups line up with the N tile's 32-channel groups
  Trace tr;
  for (long long idx = 0; idx < n_items; ++idx) {
    const Item im = decode(idx, p, th);
    const int dy = p.up > 1 ? im.tap0 / p.up : 0, dx = p.up > 1 ? im.tap0 % p.up : 0;
    for (int c = 0; c < 2; ++c) {
      long long t0 = tr.now();
      mbar_wait(smem_u32(staged + c), static_cast<uint32_t>(idx & 1));
      tr.add(kTrEwWait, t0);
      t0 = tr.now();
      if constexpr (FUSE_P) {  // P groups 2 nt, 2 nt + 1 of batch image b: 2 n_ntiles groups per image
        if (lead) tma_store4d(out_map, smem_u32(tiles + c * tile_bytes), 0, im.tx0, im.ty0 + c * 8, (im.b * p.n_ntiles + im.nt) * 2);
      } else {
        for (int blk = 0; blk < MT * NQ; ++blk) {
          const int ch0 = im.nt * N + (blk % NQ) * 32, iy0 = im.ty0 + (blk / NQ) * kTH + c * 8;
          if (ch0 >= p.cout) continue;
          const uint8_t *src = tiles + c * tile_bytes + blk * BLK;
          if (whole && ch0 + 32 <= p.cout) {
            if (!lead) continue;
            const int hc = 2 * (p.out_c0 + ch0);  // first half of the group in a pixel row
            if (p.up == 1) {
              tma_store4d(out_map, smem_u32(src), hc, im.tx0, iy0, im.b);
            } else {
              for (int y = 0; y < 8 && iy0 + y < p.oH; ++y)
                tma_store5d(out_map, smem_u32(src + y * 1024), hc, dx, im.tx0, dy, im.b * p.oH + iy0 + y);
            }
            continue;
          }
          for (int u = et; u < 128; u += kEpiThreads) {  // (row, 16-channel half)
            const int r = u >> 1, h = u & 1, iy = iy0 + (r >> 3), ix = im.tx0 + (r & 7);
            if (ch0 + 16 * h >= p.cout || iy >= p.oH || ix >= p.oW) continue;
            const int oc = p.out_c0 + ch0 + 16 * h, Y = iy * p.up + dy, X = ix * p.up + dx;
            uint8_t *op = p.out_h16 + ((static_cast<size_t>(im.b) * p.out_H + Y) * p.out_W + X) * (4 * static_cast<size_t>(p.out_C)) +
                          (oc / 32) * 128 + (oc % 32) * 2;
            const uint8_t *row = src + r * 128;
  #pragma unroll
            for (int k = 0; k < 2; ++k) {
              *reinterpret_cast<uint4 *>(op + 16 * k) = *reinterpret_cast<const uint4 *>(row + (((2 * h + k) ^ (r & 7)) << 4));
              *reinterpret_cast<uint4 *>(op + 64 + 16 * k) = *reinterpret_cast<const uint4 *>(row + (((4 + 2 * h + k) ^ (r & 7)) << 4));
            }
          }
        }
      }
      if (lead) {
        bulk_commit();
        bulk_wait_read();
      }
      mbar_arrive(smem_u32(freed + c));
      tr.add(kTrEwBusy, t0);
    }
  }
  if (lead) {
    bulk_wait_all();  // the image is written before this grid counts as complete for the next layer
    tr.flush(0);
  }
}

// FUSE_P (N = 128, MT = 1, HALO; the CenterHead's batched ConvModule conv): after the pair split the consumers also run
// the tap-as-N GEMM of the next layer, P[pixel][tap * 3 + co] = sum_c mid[pixel][c] W2[c][tap * 3 + co], on the staged
// pair rows of each of the N tile's two 64-channel heads (A: pair blocks 2j, 2j + 1; B: one extra weight-ring fill per
// item holding both heads' W2 images), and stage P over the retired pair blocks for the epilogue thread: the output
// convs' input image is never written.  The wgmma order is head_out9_kernel's, so P is bit-identical to what out9
// computes from the image read back, and p3d_head_tap_sum finishes the convs.
// RES (pair tile, up == 1): each consumer thread adds the residual of its own fragment elements, read from global memory
// (the hi and lo' halves of two adjacent channels: 4 + 4 bytes), before ReLU; the residual-free instantiations compile
// to the code they have without it.
template <int N, int MT, bool HALO, bool FUSE_P = false, bool RES = false, bool FLUSH = false>
__global__ void __launch_bounds__(kDenseThreads, 1)
    dense_conv_f16_kernel(const __grid_constant__ CUtensorMap in_map, const __grid_constant__ CUtensorMap out_map,
                          const KParams<FUSE_P, RES> p) {
  using C = Cfg<N, MT, HALO>;
  static_assert(!(FUSE_P && RES), "a residual launch writes the pixel H16 image");
  static_assert(!FUSE_P || (N == 128 && MT == 1 && HALO && 2 * kP2Bytes == C::B_BYTES &&
                            2 * 64 * kPPitch * 4 <= C::PAIR_BYTES),
                "fused P: two 64-channel heads' W2 images fill one weight slot; P fits over the pair blocks");
  constexpr int TH = kTH * MT;  // output tile height
  constexpr int H = N / 2;      // accumulator registers of the hi products of one M tile; the cross products follow
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");  // the input image is the previous layer's output
  const int up2 = p.up * p.up;
  const long long n_total = static_cast<long long>(p.B) * p.tiles_y * p.tiles_x * p.n_ntiles * (p.up > 1 ? up2 : 1);
  if (static_cast<long long>(blockIdx.x) >= n_total) return;
  const long long n_items = (n_total - blockIdx.x + gridDim.x - 1) / gridDim.x;  // round robin: see decode

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // full barriers: one producer arrive + the bytes of the load; empty barriers: one arrive per consumer warp once the
  // wgmma that read the slot have retired.  Activation full[NA] | empty[NA] | weight full[NB] | empty[NB] | staging
  // tile of consumer c staged[2] (one arrive per consumer thread) | free[2] (one arrive per epilogue thread).
  __shared__ __align__(8) unsigned long long s_bar[2 * kMaxA + 2 * kMaxB + 4];
  constexpr int kAF = 0, kAE = kMaxA, kBF = 2 * kMaxA, kBE = 2 * kMaxA + kMaxB, kSS = 2 * kMaxA + 2 * kMaxB, kSF = kSS + 2;

  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127;
  if (tid == 0) {
    for (int s = 0; s < C::NA; ++s) {
      mbar_init(smem_u32(&s_bar[kAF + s]), 1);
      mbar_init(smem_u32(&s_bar[kAE + s]), kConsumerWarps);
    }
    for (int s = 0; s < C::NB; ++s) {
      mbar_init(smem_u32(&s_bar[kBF + s]), 1);
      mbar_init(smem_u32(&s_bar[kBE + s]), kConsumerWarps);
    }
    for (int c = 0; c < 2; ++c) {
      mbar_init(smem_u32(&s_bar[kSS + c]), 128);
      mbar_init(smem_u32(&s_bar[kSF + c]), kEpiThreads);
    }
    fence_mbar_init();
  }
  __syncthreads();  // the only block-wide barrier: the mbarriers are initialised
  const uint32_t a_ring = smem_u32(smem);
  const uint32_t b_ring = a_ring + C::NA * C::A_BYTES;
  // staging tiles of the two consumer warpgroups, after the weight ring
  float *const stg = reinterpret_cast<float *>(smem + C::NA * C::A_BYTES + C::NB * C::B_BYTES);
  const bool pairs = p.out_nchw == nullptr;  // stage fp16-pair rows for TMA stores (epilogue_pairs)
  const int G = p.Cin / 32;
  // steps / activation units per item: HALO: one unit per group, 9 taps each; TAP: one unit per (tap, group)
  const int taps_item = p.up > 1 ? 1 : p.taps;
  const int units_item = HALO ? G : taps_item * G;
  const int steps_item = units_item * C::SPU;
  // Ring positions advance by one slot per fill / use; the phase bit flips when the slot index wraps.  The consumers wait
  // for full[slot] to complete the phase of the current pass; the producer waits for empty[slot] to complete the phase
  // of the previous pass (parity ph ^ 1: on the first pass that is the phase before the barrier's first, which counts as
  // complete, so the first NA / NB fills do not wait).

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(C::P_REGS));
    if (tid >= 32) {
      if (pairs)
        epilogue_pairs<N, MT, FUSE_P>(p, &out_map, reinterpret_cast<const uint8_t *>(stg), C::STG_WG * 4, s_bar + kSS, s_bar + kSF,
                              n_items, TH, tid - 32);
      else
        epilogue_warps<N, MT>(p, stg, s_bar + kSS, s_bar + kSF, n_items, TH, tid - 32);
      return;
    }
    // ------------------------------------------------------------------------------------------ producer
    if (tid != 0) return;
    uint32_t a_slot = 0, a_ph = 0, b_slot = 0, b_ph = 0;
    Trace tr;
    for (long long idx = 0; idx < n_items; ++idx) {
      const Item im = decode(idx, p, TH);
      const uint8_t *w_tile = p.packed_w + static_cast<size_t>(im.nt) * p.taps * (p.Cin / 16) * C::B_BLK;
      // TAP units are (tap, group) with the group fastest; dy, dx follow the tap without dividing
      int dy = 0, dx = 0;
      for (int tu = 0; tu < (HALO ? 1 : taps_item); ++tu) {
        const int tap = p.up > 1 ? im.tap0 : tu;
        for (int g = 0; g < G; ++g) {
          const uint32_t abar = smem_u32(&s_bar[kAF + a_slot]), a_dst = a_ring + a_slot * C::A_BYTES;
          const long long t0 = tr.now();
          mbar_wait(smem_u32(&s_bar[kAE + a_slot]), a_ph ^ 1u);
          tr.add(kTrAEmpty, t0);
          mbar_arrive_expect_tx(abar, static_cast<uint32_t>(C::A_ROWS * 128));
          if (HALO) {
            tma_tile4d(a_dst, &in_map, g * 64, im.tx0 - 1, im.ty0 - 1, im.b, abar);
          } else {
            const int x = im.tx0 * p.stride - p.pad + dx, y = im.ty0 * p.stride - p.pad + dy;  // may be negative: zero fill
            tma_tile4d(a_dst, &in_map, g * 64, x, y, im.b, abar);
          }
          if (++a_slot == C::NA) a_slot = 0, a_ph ^= 1u;
          for (int t = 0; t < C::SPU; ++t) {
            const uint32_t bbar = smem_u32(&s_bar[kBF + b_slot]);
            const long long t1 = tr.now();
            mbar_wait(smem_u32(&s_bar[kBE + b_slot]), b_ph ^ 1u);
            tr.add(kTrBEmpty, t1);
            mbar_arrive_expect_tx(bbar, static_cast<uint32_t>(C::B_BYTES));
            bulk_g2s(b_ring + b_slot * C::B_BYTES, w_tile + (static_cast<size_t>(HALO ? t : tap) * (p.Cin / 16) + 2 * g) * C::B_BLK,
                     static_cast<uint32_t>(C::B_BYTES), bbar);
            if (++b_slot == C::NB) b_slot = 0, b_ph ^= 1u;
          }
        }
        if (++dx == p.kw) dx = 0, ++dy;
      }
      if constexpr (FUSE_P) {  // the item's W2 images, used after its last step
        const uint32_t bbar = smem_u32(&s_bar[kBF + b_slot]);
        const long long t1 = tr.now();
        mbar_wait(smem_u32(&s_bar[kBE + b_slot]), b_ph ^ 1u);
        tr.add(kTrBEmpty, t1);
        mbar_arrive_expect_tx(bbar, static_cast<uint32_t>(C::B_BYTES));
        bulk_g2s(b_ring + b_slot * C::B_BYTES, p.packed_w2 + static_cast<size_t>(im.nt) * C::B_BYTES,
                 static_cast<uint32_t>(C::B_BYTES), bbar);
        if (++b_slot == C::NB) b_slot = 0, b_ph ^= 1u;
      }
    }
    tr.flush(0);
    return;
  }

  // -------------------------------------------------------------------------------------------- consumers
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(C::C_REGS));
  const int cw = wg - 1;                 // rows 64 cw .. 64 cw + 63 of every M tile
  const bool warp_leader = (tid & 31) == 0;
  auto release = [&](int base, uint32_t slot) {
    if (warp_leader) mbar_arrive(smem_u32(&s_bar[base + slot]));
  };
  uint32_t a_slot = 0, a_ph = 0, b_slot = 0, b_ph = 0;
  // acc: per M tile the hi x hi products since the last flush [0, H), then the cross products [H, N); tot: the hi x hi
  // products of the flushed steps.  The tensor core's own accumulation does not round to nearest and drifts over a long
  // chain, so every kFlush steps (HALO: one 32-channel group's 9 taps) the hi partial is added into tot with
  // round-to-nearest FADDs and the next step's first hi wgmma starts it over (scale_d = 0).  Only the FLUSH instantiations
  // do this, for chains longer than kFlushTerms: tot costs 32 to 64 registers (spills in the N = 128 and MT = 2 ones) and
  // every flush drains the wgmma pipeline, so the shorter chains keep the single accumulator.
  float acc[C::ACC], tot[MT * H];
  bool ovf = false;  // fp16 range overflow of the pair tile (status bit 0)
  Trace tr;
  const long long t_start = tr.now();
  for (long long idx = 0; idx < n_items; ++idx) {
#pragma unroll
    for (int i = 0; i < C::ACC; ++i) acc[i] = 0.f;
#pragma unroll
    for (int i = 0; i < MT * H; ++i) tot[i] = 0.f;
    const Item im = decode(idx, p, TH);
    // pair tile: the item's scale / shift columns are staged in shared memory while the K loop runs, in one of two
    // buffers (item parity) after the warpgroup's pair blocks; its epilogue reads them after a warpgroup barrier
    const uint32_t ss = smem_u32(stg) + cw * C::STG_WG * 4 + C::PAIR_BYTES + static_cast<uint32_t>(idx & 1) * 2 * N * 4;
    if (pairs) {
      for (int c = wtid; c < 2 * N; c += 128) {
        const int ch = im.nt * N + c % N;
        const float *src = c < N ? p.scale : p.shift;
        st_shared_u32(ss + c * 4, __float_as_uint(ch < p.cout && src ? __ldg(src + ch) : (c < N ? 1.0f : 0.0f)));
      }
    }
    // slots of the step whose wgmma group is still in flight: weight slot, and the activation slot when that step was
    // the last one of its unit (-1 otherwise)
    uint32_t prev_b = 0;
    int prev_a = -1;
    bool pending = false;
    int step = 0;             // steps of the item issued so far
    uint32_t hi_scale = 1u;   // 0: the step's first hi wgmma starts the hi partial over
    for (int ua = 0; ua < units_item; ++ua) {
      long long t0 = tr.now();
      mbar_wait(smem_u32(&s_bar[kAF + a_slot]), a_ph);
      tr.add(kTrAFull, t0);
      const uint32_t a_base = a_ring + a_slot * C::A_BYTES;
      for (int t = 0; t < C::SPU; ++t) {
        t0 = tr.now();
        mbar_wait(smem_u32(&s_bar[kBF + b_slot]), b_ph);
        tr.add(kTrBFull, t0);
        const uint32_t b_base = b_ring + b_slot * C::B_BYTES;
        wg_fence();
#pragma unroll
        for (int kb = 0; kb < 2; ++kb) {
          const uint32_t bk = b_base + static_cast<uint32_t>(kb * C::B_BLK);
          const uint64_t dbh = smem_desc(bk, 2 * N * 16, 128), dbl = smem_desc(bk + N * 16, 2 * N * 16, 128);
#pragma unroll
          for (int mt = 0; mt < MT; ++mt) {
            uint32_t a0, sbo;
            if (HALO) {  // this warpgroup's 8 image rows of M tile mt, shifted by the tap
              a0 = a_base + static_cast<uint32_t>(((mt * kTH + cw * 8 + t / 3) * kPitch + t % 3) * 128);
              sbo = kPitch * 128;
            } else {
              a0 = a_base + static_cast<uint32_t>((mt * kM + cw * 64) * 128);
              sbo = 1024;
            }
            const uint64_t dah = desc_sw128(a0 + kb * 32, sbo), dal = desc_sw128(a0 + (2 + kb) * 32, sbo);
            float *d = acc + mt * N;
            wg::mma_f16<N>(d, dah, dbh, kb == 0 ? hi_scale : 1u);  // A_hi x B_hi
            wg::mma_f16<N>(d + H, dah, dbl, 1u);  // A_hi x B_lo'
            wg::mma_f16<N>(d + H, dal, dbh, 1u);  // A_lo' x B_hi
          }
        }
        wg_commit();
        t0 = tr.now();
        const bool flush = FLUSH && ++step % kFlush == 0 && step < steps_item;
        if (flush)
          wg_wait<0>();  // this step's group has retired too: the hi partial can be read
        else
          wg_wait<1>();  // the previous step's group has retired: its slots go back to the producer
        tr.add(kTrMma, t0);
        if (flush) {
          wg_fence_acc<C::ACC>(acc);
#pragma unroll
          for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int i = 0; i < H; ++i) tot[mt * H + i] += acc[mt * N + i];
        }
        hi_scale = flush ? 0u : 1u;
        if (pending) {
          release(kBE, prev_b);
          if (prev_a >= 0) release(kAE, static_cast<uint32_t>(prev_a));
        }
        pending = true;
        prev_b = b_slot;
        prev_a = t == C::SPU - 1 ? static_cast<int>(a_slot) : -1;
        if (++b_slot == C::NB) b_slot = 0, b_ph ^= 1u;
      }
      if (++a_slot == C::NA) a_slot = 0, a_ph ^= 1u;
    }
    long long t0 = tr.now();
    wg_wait<0>();
    tr.add(kTrMma, t0);
    t0 = tr.now();
    release(kBE, prev_b);
    release(kAE, static_cast<uint32_t>(prev_a));  // the item's last step ends a unit
    wg_fence_acc<C::ACC>(acc);
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int i = 0; i < H; ++i) acc[mt * N + i] += tot[mt * H + i];  // the last partial joins the total
    // fill this warpgroup's staging tile once the epilogue warps have drained the previous item from it, and go on with
    // the next item
    tr.add(kTrEpi, t0);
    t0 = tr.now();
    if (idx > 0) mbar_wait(smem_u32(&s_bar[kSF + cw]), static_cast<uint32_t>((idx - 1) & 1));
    tr.add(kTrStageFree, t0);
    t0 = tr.now();
    if (pairs) {
      // fp16-pair rows, the operations of epilogue_warps in its order: per 8-column group j, lanes 4q .. 4q + 3 write
      // the hi and the lo' 16-byte chunks of fragment row q (mod 8), which the swizzle puts on distinct banks
      const int lane = wtid & 31, key = lane >> 2;  // fragment row & 7
      // shared address of fragment row q, column pair (lane & 3) of chunk jj's hi / lo' halves; the (M tile, group)
      // block and the row half h are immediate offsets
      const uint32_t row = smem_u32(stg) + cw * C::STG_WG * 4 + ((wtid >> 5) * 16 + key) * 128 + (lane & 3) * 4;
      uint32_t a_hi[4], a_lo[4];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) a_hi[jj] = row + ((jj ^ key) << 4), a_lo[jj] = row + (((4 + jj) ^ key) << 4);
      // the scale / shift columns are staged once the warpgroup passes its barrier; the barrier's zero output makes the
      // reads depend on it
      uint32_t after_bar;
      asm volatile("bar.sync %1, 128;\n\tmov.u32 %0, 0;" : "=r"(after_bar) : "r"(1 + cw) : "memory");
      const uint32_t sc_col = ss + after_bar + (lane & 3) * 8;
      // RES: fragment row q + 8 h of M tile mt is pixel (iy + mt * kTH + h, ix); column pair (lane & 3) of 8-column group
      // j is channel nt * N + 8 j + 2 (lane & 3), at byte (channel / 32) * 128 + (channel % 32) * 2 of a residual row
      // (+ 64 for lo').  r_off: byte offset of that pixel's first column pair in the residual image (< 2^31, checked by
      // the host), -1 outside the output; r_rem: channels of the N tile below cout
      int r_off[MT][2], r_rem = 0;
      if constexpr (RES) {
        const int r_iy = im.ty0 + cw * 8 + (wtid >> 5) * 2, r_ix = im.tx0 + key;
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int Y = r_iy + mt * kTH + h;
            r_off[mt][h] = r_ix < p.oW && Y < p.oH
                               ? ((im.b * p.out_H + Y) * p.out_W + r_ix) * 4 * p.res_C + (im.nt * N / 32) * 128 + (lane & 3) * 4
                               : -1;
          }
        r_rem = p.cout - im.nt * N;
      }
      bool o[MT][2] = {};
#pragma unroll
      for (int j = 0; j < N / 8; ++j) {
        // columns past cout: scale 1, shift 0, value 0, no overflow
        const float2 sc = ld_shared_f2(sc_col + j * 32), sh = ld_shared_f2(sc_col + (N + j * 8) * 4);
        const float sc0 = sc.x, sc1 = sc.y, sh0 = sh.x, sh1 = sh.y;
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int i = j * 4 + h * 2;
            float v0 = fmaf(acc[mt * N + H + i], kLoInv, acc[mt * N + i]);
            float v1 = fmaf(acc[mt * N + H + i + 1], kLoInv, acc[mt * N + i + 1]);
            v0 = fmaf(v0, sc0, sh0);
            v1 = fmaf(v1, sc1, sh1);
            if constexpr (RES) {
              // pixels outside the output and channels past cout are not stored: no residual read there
              if (r_off[mt][h] >= 0 && j * 8 < r_rem) {
                const uint8_t *rp = p.res_h16 + r_off[mt][h] + (j / 4) * 128 + (j & 3) * 16;
                const uint32_t rh = __ldg(reinterpret_cast<const unsigned int *>(rp));
                const uint32_t rl = __ldg(reinterpret_cast<const unsigned int *>(rp + 64));
                const float2 fh = __half22float2(*reinterpret_cast<const __half2 *>(&rh));
                const float2 fl = __half22float2(*reinterpret_cast<const __half2 *>(&rl));
                v0 += fmaf(fl.x, kLoInv, fh.x);
                v1 += fmaf(fl.y, kLoInv, fh.y);
              }
            }
            if (p.relu) v0 = fmaxf(v0, 0.f), v1 = fmaxf(v1, 0.f);
            __half2 hi, lo;
            split_h16x2(v0, v1, hi, lo, o[mt][h]);
            const uint32_t off = (mt * (N / 32) + j / 4) * C::PAIR_BLK + h * 8 * 128;
            st_shared_u32(a_hi[j & 3] + off, *reinterpret_cast<const uint32_t *>(&hi));
            st_shared_u32(a_lo[j & 3] + off, *reinterpret_cast<const uint32_t *>(&lo));
          }
        }
      }
      // only values that reach the image count (fragment row q + 8 h: pixel row iy + h, column ix)
      const int iy = im.ty0 + cw * 8 + (wtid >> 5) * 2, ix = im.tx0 + key;
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
        ovf |= ix < p.oW && ((o[mt][0] && iy + mt * kTH < p.oH) || (o[mt][1] && iy + mt * kTH + 1 < p.oH));
      fence_proxy_async();  // the TMA stores (FUSE_P: the wgmma) read the tile through the async proxy
      if constexpr (FUSE_P) {
        asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");  // the warpgroup's pair rows are all staged
        const long long t1 = tr.now();
        mbar_wait(smem_u32(&s_bar[kBF + b_slot]), b_ph);
        tr.add(kTrBFull, t1);
        const uint32_t w2 = b_ring + b_slot * C::B_BYTES, tile = smem_u32(stg) + cw * C::STG_WG * 4;
        float pacc[64];  // per head j: hi products [32 j, 32 j + 16), cross products [32 j + 16, 32 j + 32)
#pragma unroll
        for (int i = 0; i < 64; ++i) pacc[i] = 0.f;
        wg_fence();
#pragma unroll
        for (int j = 0; j < 2; ++j) {
#pragma unroll
          for (int k = 0; k < 2; ++k) {  // 32-channel group of the head, then k-step: head_out9_kernel's order
#pragma unroll
            for (int kb = 0; kb < 2; ++kb) {
              const uint32_t bk = w2 + static_cast<uint32_t>(j * kP2Bytes + (k * 2 + kb) * kP2Blk);
              const uint64_t dbh = smem_desc(bk, 2 * 32 * 16, 128), dbl = smem_desc(bk + 32 * 16, 2 * 32 * 16, 128);
              const uint32_t a0 = tile + static_cast<uint32_t>((2 * j + k) * C::PAIR_BLK);
              const uint64_t dah = desc_sw128(a0 + kb * 32), dal = desc_sw128(a0 + (2 + kb) * 32);
              wg::mma_f16<32>(pacc + 32 * j, dah, dbh, 1u);
              wg::mma_f16<32>(pacc + 32 * j + 16, dah, dbl, 1u);
              wg::mma_f16<32>(pacc + 32 * j + 16, dal, dbh, 1u);
            }
          }
        }
        wg_commit();
        wg_wait<0>();
        release(kBE, b_slot);
        if (++b_slot == C::NB) b_slot = 0, b_ph ^= 1u;
        wg_fence_acc<64>(pacc);
        asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");  // every warp's wgmma have read the pair rows
        // P[group j][row][col] = hi + cross * 2^-11 over the retired pair blocks, columns 0 .. kPPitch - 1 (27 is 0)
        float *const pt = stg + cw * C::STG_WG;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
#pragma unroll
          for (int i = 0; i < 16; i += 2) {
            const int r = frag_row(i, wtid), c = frag_col(i, wtid);
            if (c < kPPitch)
              *reinterpret_cast<float2 *>(pt + (j * 64 + r) * kPPitch + c) =
                  make_float2(fmaf(pacc[32 * j + 16 + i], kLoInv, pacc[32 * j + i]),
                              fmaf(pacc[32 * j + 17 + i], kLoInv, pacc[32 * j + 1 + i]));
          }
        }
        fence_proxy_async();
      }
    } else {
      // hi + cross * 2^-11 in fp32, row mt * 64 + fragment row
      float *const st = stg + cw * C::STG_WG;
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
        for (int i = 0; i < H; i += 2) {
          const int r = mt * 64 + frag_row(i, wtid), c = frag_col(i, wtid);
          *reinterpret_cast<float2 *>(st + r * C::SP + c) =
              make_float2(fmaf(acc[mt * N + H + i], kLoInv, acc[mt * N + i]), fmaf(acc[mt * N + H + i + 1], kLoInv, acc[mt * N + i + 1]));
        }
      }
    }
    mbar_arrive(smem_u32(&s_bar[kSS + cw]));
    tr.add(kTrEpi, t0);
  }
  if (ovf && p.status) atomicOr(p.status, 1);
  if (cw == 0) {
    tr.count(kTrItems, static_cast<unsigned long long>(n_items));
    tr.add(kTrCycles, t_start);
  }
  if (wtid == 0) tr.flush(cw);
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
  out[q] = merge_h16(grp[c % 32], grp[32 + c % 32]);
}

using Encode = CUresult (*)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                            const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                            CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline Encode tensor_map_encoder() {  // cuTensorMapEncodeTiled from the driver, or null
  static Encode encode = nullptr;
  if (!encode) {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) != cudaSuccess || !fn) return nullptr;
    encode = reinterpret_cast<Encode>(fn);
  }
  return encode;
}

inline int make_image_map(const void *img, int B, int H, int W, int Cin, int stride, int box_x, int box_y, CUtensorMap *map) {
  // Cin = channels per pixel of the image in memory
  const Encode encode = tensor_map_encoder();
  if (!encode) return P3D_ERR_UNSUPPORTED;
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

// Store map of the pair-tile epilogue over the out_C-channel output image.  Convolution: {2 out_C halfs, out_W, out_H, B}
// with an 8 x 8-pixel box of one 32-channel group.  Transposed conv (kernel = stride = up, input H x W): the output
// pixel (iy up + dy, ix up + dx) as {2 out_C halfs, up (dx), W (ix), up (dy), B H (iy)} with a box of one tap's 8 pixels
// of an input row.  Boxes past the right and bottom edges are clipped.
inline int make_out_map(void *img, int B, int H, int W, int out_C, int up, CUtensorMap *map) {
  const Encode encode = tensor_map_encoder();
  if (!encode) return P3D_ERR_UNSUPPORTED;
  const cuuint64_t row = static_cast<cuuint64_t>(4) * out_C;  // bytes per output pixel
  CUresult r;
  if (up == 1) {
    const cuuint64_t gdim[4] = {static_cast<cuuint64_t>(2 * out_C), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H),
                                static_cast<cuuint64_t>(B)};
    const cuuint64_t gstride[3] = {row, row * W, row * W * H};
    const cuuint32_t box[4] = {64u, static_cast<cuuint32_t>(kTW), 8u, 1u}, estride[4] = {1u, 1u, 1u, 1u};
    r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, img, gdim, gstride, box, estride, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else {
    const cuuint64_t u = static_cast<cuuint64_t>(up), ow = u * W;
    const cuuint64_t gdim[5] = {static_cast<cuuint64_t>(2 * out_C), u, static_cast<cuuint64_t>(W), u,
                                static_cast<cuuint64_t>(B) * H};
    const cuuint64_t gstride[4] = {row, row * u, row * ow, row * ow * u};
    const cuuint32_t box[5] = {64u, 1u, static_cast<cuuint32_t>(kTW), 1u, 1u}, estride[5] = {1u, 1u, 1u, 1u, 1u};
    r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, img, gdim, gstride, box, estride, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  return r == CUDA_SUCCESS ? P3D_OK : P3D_ERR_INVALID_ARG;
}

// Store map of the FUSE_P epilogue over the P buffer [B * p_groups][H][W][kPPitch] fp32: one box is an item's two
// groups of one consumer warpgroup's 8 x 8 pixels; boxes past the right and bottom edges are clipped.
inline int make_p_map(float *pbuf, int B, int H, int W, int p_groups, CUtensorMap *map) {
  const Encode encode = tensor_map_encoder();
  if (!encode) return P3D_ERR_UNSUPPORTED;
  const cuuint64_t px = static_cast<cuuint64_t>(4) * kPPitch;  // bytes per pixel of a group
  const cuuint64_t gdim[4] = {static_cast<cuuint64_t>(kPPitch), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H),
                              static_cast<cuuint64_t>(B) * p_groups};
  const cuuint64_t gstride[3] = {px, px * W, px * W * H};
  const cuuint32_t box[4] = {static_cast<cuuint32_t>(kPPitch), static_cast<cuuint32_t>(kTW), 8u, 2u}, estride[4] = {1u, 1u, 1u, 1u};
  const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, pbuf, gdim, gstride, box, estride, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? P3D_OK : P3D_ERR_INVALID_ARG;
}

template <int N, int MT, bool HALO, bool FUSE_P = false, bool RES = false>
int launch(const CUtensorMap &map, const CUtensorMap &out_map, const KParams<FUSE_P, RES> &p, cudaStream_t st) {
  using C = Cfg<N, MT, HALO>;
  const size_t smem = static_cast<size_t>(C::NA) * C::A_BYTES + static_cast<size_t>(C::NB) * C::B_BYTES + C::STG_BYTES + 1024;
  if (smem > static_cast<size_t>(kSmemBudget)) return P3D_ERR_UNSUPPORTED;
  // a chain of more than kFlushTerms products per output drifts in one wgmma accumulator: the FLUSH instantiation
  const bool flush = static_cast<long long>(p.Cin) * (p.up > 1 ? 1 : p.taps) > kFlushTerms;
  auto kern = flush ? dense_conv_f16_kernel<N, MT, HALO, FUSE_P, RES, !FUSE_P> : dense_conv_f16_kernel<N, MT, HALO, FUSE_P, RES>;
  P3D_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  const long long work = static_cast<long long>(p.B) * p.tiles_y * p.tiles_x * p.n_ntiles * (p.up > 1 ? p.up * p.up : 1);
  cudaLaunchConfig_t cfg = {};
  const long long sms = num_sms();
  cfg.gridDim = dim3(static_cast<unsigned int>(work < sms ? work : sms));
  cfg.blockDim = dim3(kDenseThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  P3D_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, map, out_map, p));
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// CenterHead output convs with the 9 taps in the N dimension ("tap-as-N", center_head.py:80-117 SeparateHead finals).
//
// A 3x3 conv with <= 3 output channels would be 9 * Cin/16 k-steps of N = 16 MMAs per 128 pixels as an ordinary conv.
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

// Spatial half of the fused output convs (FUSE_P): out[b][plane0 + co][y][x] = bias + sum_tap P[y + dy][x + dx][tap * 3
// + co], taps in out9's order with +0 for neighbours outside the image (what out9 adds there from its zero-filled
// halo), so the planes are bit-identical to out9's.  A block stages the 10 x 34 haloed pixels of one 8 x 32 output tile
// of one P group with coalesced 16-byte loads (row pitch 27 floats: the per-pixel reads of a warp hit distinct banks);
// one thread per output pixel, so a warp stores 32 consecutive floats of a plane row.
namespace tapsum {
constexpr int kTX = 32, kTY = 8, kThreads = kTX * kTY, kSX = kTX + 2, kSY = kTY + 2, kSP = 27;

struct Params {
  int B, H, W, groups, planes, tiles_x, tiles_y;
  const float *p;               // [B * groups][H][W][kPPitch]
  const float *bias;            // [groups][4]
  const int32_t *plane0, *cnt;  // [groups]
  float *out;                   // [B, planes, H, W]
};

__global__ void __launch_bounds__(kThreads) head_tap_sum_kernel(const Params p) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  __shared__ float s_p[kSY * kSX * kSP];
  long long q = blockIdx.x;
  const int tx0 = static_cast<int>(q % p.tiles_x) * kTX;
  q /= p.tiles_x;
  const int ty0 = static_cast<int>(q % p.tiles_y) * kTY;
  q /= p.tiles_y;
  const int g = static_cast<int>(q % p.groups), b = static_cast<int>(q / p.groups);
  const float *src = p.p + static_cast<size_t>(b * p.groups + g) * p.H * p.W * kPPitch;
  constexpr int V = kPPitch / 4;  // float4 per pixel
  for (int u = threadIdx.x; u < kSY * kSX * V; u += kThreads) {
    const int pix = u / V, v = u - pix * V, sy = pix / kSX, sx = pix - sy * kSX, Y = ty0 - 1 + sy, X = tx0 - 1 + sx;
    float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
    if (Y >= 0 && Y < p.H && X >= 0 && X < p.W)
      f = __ldg(reinterpret_cast<const float4 *>(src + (static_cast<size_t>(Y) * p.W + X) * kPPitch) + v);
    float *d = s_p + pix * kSP + v * 4;
    d[0] = f.x;
    d[1] = f.y;
    d[2] = f.z;
    if (v < V - 1) d[3] = f.w;  // column 27 is not used
  }
  __syncthreads();
  const int lx = threadIdx.x % kTX, ly = threadIdx.x / kTX, X = tx0 + lx, Y = ty0 + ly;
  if (X >= p.W || Y >= p.H) return;
  const int cnt = __ldg(p.cnt + g), p0 = __ldg(p.plane0 + g);
  const size_t plane = static_cast<size_t>(p.H) * p.W;
  float *op = p.out + (static_cast<size_t>(b) * p.planes + p0) * plane + static_cast<size_t>(Y) * p.W + X;
  for (int co = 0; co < cnt; ++co) {
    float s = __ldg(p.bias + g * 4 + co);
#pragma unroll
    for (int t = 0; t < 9; ++t) s += s_p[((ly + t / 3) * kSX + lx + t % 3) * kSP + t * 3 + co];
    op[co * plane] = s;
  }
}
}  // namespace tapsum

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

#ifdef P3D_DENSE_TRACE
// Trace build only (not in p3d_b200.h): copies the per-CTA sums of dcf::TraceField ([max_ctas][fields] uint64) to the
// host and zeroes them when reset != 0.  Returns the number of fields per CTA.
extern "C" int p3d_dense_trace_read(unsigned long long *host, int max_ctas, int reset) {
  const size_t n = static_cast<size_t>(max_ctas < dcf::kTrMaxCtas ? max_ctas : dcf::kTrMaxCtas) * dcf::kTrFields;
  P3D_CUDA_CHECK(cudaDeviceSynchronize());
  if (host) P3D_CUDA_CHECK(cudaMemcpyFromSymbol(host, dcf::g_dense_trace, n * sizeof(unsigned long long)));
  if (reset) {
    void *dev = nullptr;
    P3D_CUDA_CHECK(cudaGetSymbolAddress(&dev, dcf::g_dense_trace));
    P3D_CUDA_CHECK(cudaMemset(dev, 0, sizeof(dcf::g_dense_trace)));
    P3D_CUDA_CHECK(cudaDeviceSynchronize());
  }
  return dcf::kTrFields;
}
#endif

// packed weights: per N tile the image p3d_sparse_conv_f16_pack_weights makes of W[tap][Cin][n_tile] (zero-padded columns)
extern "C" size_t p3d_dense_conv2d_f16_packed_weight_bytes(int taps, int Cin, int Cout, int n_tile) {
  if (taps < 1 || Cin < 32 || Cin % 32 || Cout < 1 || (n_tile != 16 && n_tile != 32 && n_tile != 64 && n_tile != 128)) return 0;
  const size_t tiles = static_cast<size_t>((Cout + n_tile - 1) / n_tile);
  return align_up(tiles * taps * Cin * static_cast<size_t>(n_tile) * 4);
}

namespace {
// mode: 0 auto (HALO for 3x3 stride 1 pad 1 convolutions, TAP otherwise), 1 force TAP; m_tiles: 0 auto, 1 or 2.  RES:
// res_h16 / res_C as p3d_dense_conv2d_f16_residual takes them (checked by the caller)
template <bool RES>
int dense_conv2d_f16(const void *in_h16, int B, int H, int W, int Cin, const void *packed_weight, int Cout, int n_tile, int kh,
                     int kw, int stride, int pad, int up, const float *scale, const float *shift, int relu, void *out_h16,
                     int out_C, int out_c0, float *out_nchw, const void *res_h16, int res_C, int mode, int m_tiles,
                     int32_t *status_dev, p3d_stream_t stream) {
  if (!in_h16 || !packed_weight || (!out_h16 && !out_nchw) || B < 1 || H < 1 || W < 1 || Cout < 1 || (mode != 0 && mode != 1))
    return P3D_ERR_INVALID_ARG;
  if (Cin < 32 || Cin % 32 || (n_tile != 64 && n_tile != 128)) return P3D_ERR_UNSUPPORTED;
  if (up < 1 || (up > 1 && (kh != up || kw != up || stride != up || pad != 0))) return P3D_ERR_UNSUPPORTED;
  if (up == 1 && (kh < 1 || kw < 1 || kh * kw > 32 || stride < 1 || stride > 2 || pad < 0)) return P3D_ERR_UNSUPPORTED;
  if (out_h16 && (Cout % 16 || out_C % 32 || out_c0 % 16 || out_c0 + Cout > out_C)) return P3D_ERR_INVALID_ARG;
  if ((reinterpret_cast<uintptr_t>(in_h16) & 15) || (reinterpret_cast<uintptr_t>(packed_weight) & 15) ||
      (reinterpret_cast<uintptr_t>(out_h16) & 15))
    return P3D_ERR_INVALID_ARG;
  dcf::KParams<false, RES> p;
  if constexpr (RES) {
    p.res_h16 = static_cast<const uint8_t *>(res_h16);
    p.res_C = res_C;
  }
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
  p.n_ntiles = (Cout + n_tile - 1) / n_tile;
  p.cout = Cout;
  p.out_C = out_C;
  p.out_c0 = out_c0;
  p.relu = relu;
  p.packed_w = static_cast<const uint8_t *>(packed_weight);
  p.scale = scale;
  p.shift = shift;
  p.out_h16 = static_cast<uint8_t *>(out_h16);
  p.out_nchw = out_nchw;
  p.status = status_dev;
  const bool halo = mode == 0 && up == 1 && kh == 3 && kw == 3 && stride == 1 && pad == 1;
  // one or two M tiles per item for the narrow N <= 64 layers (N = 128 keeps one: register budget): the persistent grid
  // runs ceil(items / SMs) rounds of items MT M tiles long, so pick the MT with the fewer M-tile rounds; on a tie two M
  // tiles, which share every weight block (half the weight traffic per flop)
  int mt = m_tiles;
  if (mt != 1 && mt != 2) {
    const long long tx = (p.oW + dcf::kTW - 1) / dcf::kTW, sms = num_sms();
    const long long per_row = static_cast<long long>(B) * tx * p.n_ntiles * (up > 1 ? up * up : 1);
    const long long items1 = per_row * ((p.oH + dcf::kTH - 1) / dcf::kTH), items2 = per_row * ((p.oH + 2 * dcf::kTH - 1) / (2 * dcf::kTH));
    mt = (n_tile <= 64 && 2 * ((items2 + sms - 1) / sms) <= (items1 + sms - 1) / sms) ? 2 : 1;
  }
  if (n_tile > 64) mt = 1;  // two M tiles of a 128-wide N tile would need 256 accumulator registers per thread
  p.tiles_x = (p.oW + dcf::kTW - 1) / dcf::kTW;
  p.tiles_y = (p.oH + dcf::kTH * mt - 1) / (dcf::kTH * mt);
  CUtensorMap map;
  const int bx = halo ? dcf::kPitch : dcf::kTW, by = halo ? dcf::kTH * mt + 2 : dcf::kTH * mt;
  int rc = dcf::make_image_map(in_h16, B, H, W, Cin, p.stride, bx, by, &map);
  if (rc != P3D_OK) return rc;
  CUtensorMap omap = {};  // read only by the pair-tile epilogue of launches without fp32 planes
  if (!out_nchw && (rc = dcf::make_out_map(out_h16, B, p.oH, p.oW, out_C, up, &omap)) != P3D_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (n_tile == 128)
    return halo ? dcf::launch<128, 1, true, false, RES>(map, omap, p, st) : dcf::launch<128, 1, false, false, RES>(map, omap, p, st);
  if (mt == 2)
    return halo ? dcf::launch<64, 2, true, false, RES>(map, omap, p, st) : dcf::launch<64, 2, false, false, RES>(map, omap, p, st);
  return halo ? dcf::launch<64, 1, true, false, RES>(map, omap, p, st) : dcf::launch<64, 1, false, false, RES>(map, omap, p, st);
}
}  // namespace

extern "C" int p3d_dense_conv2d_f16(const void *in_h16, int B, int H, int W, int Cin, const void *packed_weight, int Cout,
                                    int n_tile, int kh, int kw, int stride, int pad, int up, const float *scale,
                                    const float *shift, int relu, void *out_h16, int out_C, int out_c0, float *out_nchw,
                                    int mode, int m_tiles, int32_t *status_dev, p3d_stream_t stream) {
  return dense_conv2d_f16<false>(in_h16, B, H, W, Cin, packed_weight, Cout, n_tile, kh, kw, stride, pad, up, scale, shift, relu,
                                 out_h16, out_C, out_c0, out_nchw, nullptr, 0, mode, m_tiles, status_dev, stream);
}

// p3d_dense_conv2d_f16 with a residual added before ReLU (ResNet BasicBlock conv2): pixel H16 res_h16 [B, oH, oW, res_C]
extern "C" int p3d_dense_conv2d_f16_residual(const void *in_h16, int B, int H, int W, int Cin, const void *packed_weight,
                                             int Cout, int n_tile, int kh, int kw, int stride, int pad, int up,
                                             const float *scale, const float *shift, int relu, void *out_h16, int out_C,
                                             int out_c0, float *out_nchw, const void *res_h16, int res_C, int mode,
                                             int m_tiles, int32_t *status_dev, p3d_stream_t stream) {
  if (!res_h16 || (reinterpret_cast<uintptr_t>(res_h16) & 15)) return P3D_ERR_INVALID_ARG;
  if (up != 1 || out_nchw || !out_h16 || out_c0 % 32 || res_C % 32) return P3D_ERR_UNSUPPORTED;
  if (res_C < Cout) return P3D_ERR_INVALID_ARG;
  // the kernel addresses the residual with 32-bit byte offsets
  const long long oh = (H + 2 * pad - kh) / (stride > 0 ? stride : 1) + 1, ow = (W + 2 * pad - kw) / (stride > 0 ? stride : 1) + 1;
  if (static_cast<long long>(B) * oh * ow * 4 * res_C > 0x7fffffffll) return P3D_ERR_UNSUPPORTED;
  return dense_conv2d_f16<true>(in_h16, B, H, W, Cin, packed_weight, Cout, n_tile, kh, kw, stride, pad, up, scale, shift, relu,
                                out_h16, out_C, out_c0, out_nchw, res_h16, res_C, mode, m_tiles, status_dev, stream);
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
  if (Cin < 32 || Cin % 32) return P3D_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(in_h16) & 15) || (reinterpret_cast<uintptr_t>(packed_weight) & 15) ||
      (reinterpret_cast<uintptr_t>(bias) & 15))
    return P3D_ERR_INVALID_ARG;
  namespace o9 = dcf::out9;
  // activation ring: as many slots as the shared-memory budget leaves after the alignment slack, P and the weight ring
  // (Cin = 32 / 64 / 128: 5 / 5 / 4 slots; fewer than two above Cin = 320)
  const long long w_ring = static_cast<long long>(o9::kNW) * 2 * (Cin / 32) * o9::kWBlk;
  const long long na = (dcf::kSmemBudget - 1024 - o9::kPBytes - w_ring) / o9::kABytes;
  if (na < 2) return P3D_ERR_UNSUPPORTED;
  o9::Params p;
  p.B = B;
  p.H = H;
  p.W = W;
  p.G = Cin / 32;
  p.tiles_x = (W + o9::kOT - 1) / o9::kOT;
  p.tiles_y = (H + o9::kOT - 1) / o9::kOT;
  p.groups = groups;
  p.planes = planes;
  p.NA = static_cast<int>(na < o9::kMaxNA ? na : o9::kMaxNA);
  p.packed_w = static_cast<const uint8_t *>(packed_weight);
  p.bias = bias;
  p.cin0 = cin0_dev;
  p.plane0 = plane0_dev;
  p.cnt = cnt_dev;
  p.out = out_nchw;
  CUtensorMap map;
  const int rc = dcf::make_image_map(in_h16, B, H, W, in_C, 1, o9::kHT, o9::kHT, &map);
  if (rc != P3D_OK) return rc;
  const size_t smem = static_cast<size_t>(p.NA) * o9::kABytes + static_cast<size_t>(w_ring) + o9::kPBytes + 1024;
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

// CenterHead ConvModule conv (3x3, pad 1, scale / shift, ReLU) of Cout / 64 heads fused with the GEMM of their output
// convs (dcf::dense_conv_f16_kernel<128, 1, true, true>): writes P [B][Cout / 64][H][W][28] fp32 instead of the heads'
// pixel H16 image; p3d_head_tap_sum makes the planes.
extern "C" int p3d_head_conv_p_f16(const void *in_h16, int B, int H, int W, int Cin, const void *packed_weight, int Cout,
                                   const float *scale, const float *shift, const void *packed_w2, float *p_out,
                                   int32_t *status_dev, p3d_stream_t stream) {
  if (!in_h16 || !packed_weight || !packed_w2 || !p_out || B < 1 || H < 1 || W < 1 || Cout < 1) return P3D_ERR_INVALID_ARG;
  if (Cin < 32 || Cin % 32 || Cout % 128) return P3D_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(in_h16) & 15) || (reinterpret_cast<uintptr_t>(packed_weight) & 15) ||
      (reinterpret_cast<uintptr_t>(packed_w2) & 15) || (reinterpret_cast<uintptr_t>(p_out) & 15))
    return P3D_ERR_INVALID_ARG;
  dcf::ParamsP p = {};
  p.B = B;
  p.H = p.oH = p.out_H = H;
  p.W = p.oW = p.out_W = W;
  p.Cin = Cin;
  p.taps = 9;
  p.kw = 3;
  p.stride = p.pad = p.up = 1;
  p.n_ntiles = Cout / 128;
  p.cout = Cout;
  p.relu = 1;
  p.packed_w = static_cast<const uint8_t *>(packed_weight);
  p.scale = scale;
  p.shift = shift;
  p.status = status_dev;
  p.packed_w2 = static_cast<const uint8_t *>(packed_w2);
  p.tiles_x = (W + dcf::kTW - 1) / dcf::kTW;
  p.tiles_y = (H + dcf::kTH - 1) / dcf::kTH;
  CUtensorMap map, pmap;
  int rc = dcf::make_image_map(in_h16, B, H, W, Cin, 1, dcf::kPitch, dcf::kTH + 2, &map);
  if (rc != P3D_OK || (rc = dcf::make_p_map(p_out, B, H, W, Cout / 64, &pmap)) != P3D_OK) return rc;
  return dcf::launch<128, 1, true, true>(map, pmap, p, static_cast<cudaStream_t>(stream));
}

// Output convs of p3d_head_conv_p_f16's heads from P: group g writes cnt[g] <= 3 planes from plane0[g] of out_nchw
// [B, planes, H, W] (device int32 arrays); bias [groups][4].
extern "C" int p3d_head_tap_sum(const float *p_in, int B, int H, int W, int groups, const float *bias, const int32_t *plane0_dev,
                                const int32_t *cnt_dev, int planes, float *out_nchw, p3d_stream_t stream) {
  if (!p_in || !bias || !plane0_dev || !cnt_dev || !out_nchw || B < 1 || H < 1 || W < 1 || groups < 1 || planes < 1 ||
      (reinterpret_cast<uintptr_t>(p_in) & 15))
    return P3D_ERR_INVALID_ARG;
  namespace ts = dcf::tapsum;
  ts::Params p;
  p.B = B;
  p.H = H;
  p.W = W;
  p.groups = groups;
  p.planes = planes;
  p.tiles_x = (W + ts::kTX - 1) / ts::kTX;
  p.tiles_y = (H + ts::kTY - 1) / ts::kTY;
  p.p = p_in;
  p.bias = bias;
  p.plane0 = plane0_dev;
  p.cnt = cnt_dev;
  p.out = out_nchw;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned int>(static_cast<long long>(B) * groups * p.tiles_y * p.tiles_x));
  cfg.blockDim = dim3(ts::kThreads);
  cfg.stream = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  P3D_CUDA_CHECK(cudaLaunchKernelEx(&cfg, ts::head_tap_sum_kernel, p));
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
