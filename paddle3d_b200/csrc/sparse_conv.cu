// Sparse 3-D convolution for sm_90a: rulebook build + output-stationary gather-GEMM.
//
// Replaces what SparseResNet3D asks of paddle.sparse.nn (sparse_resnet.py:31-60,84-111,125-206):
// Paddle's phi kernels build a pair list per kernel offset and run K rounds of
// gather -> cuBLAS GEMM -> scatter-add through HBM.  Here a conv is ONE kernel over an
// output-stationary neighbour map nbr[n_out, K] (row of the input feeding tap k of output o, or -1):
//
//     out[o, :] = act( (sum_k in[nbr[o][k], :] @ W[k]) * scale + shift (+ residual[o, :]) )
//
// so every output row is written once, the sum over taps runs in a fixed order (bit-reproducible
// regardless of row numbering), BatchNorm(eval)/bias/residual/ReLU are fused in the epilogue, and
// the map is built once per stage and shared by all SubM layers of the stage (the reference's
// `key='resN'`, sparse_resnet.py:44,130-158).
//
// Rulebook build = open-addressing hash of the active coordinates (64-bit entries
// (linear cell << 32 | row)), all counts kept on the device.
//
// This file holds the fp32 CUDA-core GEMM path (exact fp32 FMA accumulation, used for parity and
// for the 5-channel input layer); the wgmma 3xTF32 path lives in sparse_conv_tc.cu.
#include <cuda_fp16.h>

#include <algorithm>

#include "common.cuh"
#include "h16.cuh"

namespace p3d {
namespace {

constexpr unsigned long long kEmpty = ~0ull;

struct Dims {
  int B, D, H, W;          // input spatial
  int kd, kh, kw;          // kernel
  int sd, sh, sw;          // stride
  int pd, ph, pw;          // padding
  int oD, oH, oW;          // output spatial
};

__device__ __forceinline__ uint32_t lin(int b, int z, int y, int x, int D, int H, int W) {
  return ((static_cast<uint32_t>(b) * D + z) * H + y) * W + x;
}

__device__ __forceinline__ int lookup(const unsigned long long *__restrict__ tab, uint32_t mask, uint32_t shift,
                                      uint32_t key) {
  uint32_t h = hash32(key) >> shift;
  while (true) {
    const unsigned long long e = tab[h];
    if (e == kEmpty) return -1;
    if (static_cast<uint32_t>(e >> 32) == key) {
      const uint32_t row = static_cast<uint32_t>(e);
      return row >= 0x7fffffffu ? -1 : static_cast<int>(row);  // a site beyond the capacity or not numbered yet: no row
    }
    h = (h + 1) & mask;
  }
}

__global__ void __launch_bounds__(256) rb_insert_kernel(const int32_t *__restrict__ coords,
                                                        const int32_t *__restrict__ n_dev, int n_cap, Dims d,
                                                        unsigned long long *__restrict__ tab, uint32_t mask,
                                                        uint32_t shift) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = n_dev ? min(n_dev[0], n_cap) : n_cap;
  if (i >= n) return;
  const int4 c = *reinterpret_cast<const int4 *>(coords + static_cast<size_t>(i) * 4);
  if (c.x < 0 || c.x >= d.B || c.y < 0 || c.y >= d.D || c.z < 0 || c.z >= d.H || c.w < 0 || c.w >= d.W) return;
  const uint32_t key = lin(c.x, c.y, c.z, c.w, d.D, d.H, d.W);
  const unsigned long long want = (static_cast<unsigned long long>(key) << 32) | static_cast<uint32_t>(i);
  uint32_t h = hash32(key) >> shift;
  while (true) {
    unsigned long long cur = tab[h];
    if (cur == kEmpty) {
      cur = atomicCAS(&tab[h], kEmpty, want);
      if (cur == kEmpty) return;
    }
    if (static_cast<uint32_t>(cur >> 32) == key) {
      atomicMax(&tab[h], want);  // duplicate coordinate: the later row wins
      return;
    }
    h = (h + 1) & mask;
  }
}

// SubM map: nbr[i][k] = row of the input at  coord(i) - pad + k   (pad k/2; the centre tap is row i itself)
__global__ void __launch_bounds__(256) rb_neighbors_kernel(const int32_t *__restrict__ coords,
                                                           const int32_t *__restrict__ n_dev, long long n_cap, Dims d,
                                                           const unsigned long long *__restrict__ tab, uint32_t mask,
                                                           uint32_t shift, int32_t *__restrict__ nbr) {
  const int K = d.kd * d.kh * d.kw;
  const long long n = n_dev ? min(static_cast<long long>(n_dev[0]), n_cap) : n_cap;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  // persistent grid-stride loop: the grid is sized for the SMs, not for the (much larger) capacity
  for (long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; q < n * K; q += stride) {
    const int o = static_cast<int>(q / K), k = static_cast<int>(q - static_cast<long long>(o) * K);
    const int4 c = *reinterpret_cast<const int4 *>(coords + static_cast<size_t>(o) * 4);
    const int kz = k / (d.kh * d.kw), ky = (k / d.kw) % d.kh, kx = k % d.kw;
    const int iz = c.y - d.pd + kz, iy = c.z - d.ph + ky, ix = c.w - d.pw + kx;
    int r = -1;
    if (kz == d.kd / 2 && ky == d.kh / 2 && kx == d.kw / 2) {
      r = o;
    } else if (iz >= 0 && iz < d.D && iy >= 0 && iy < d.H && ix >= 0 && ix < d.W) {
      r = lookup(tab, mask, shift, lin(c.x, iz, iy, ix, d.D, d.H, d.W));
    }
    nbr[q] = r;
  }
}

// Strided conv: output site o of input row coord c under tap k, where c = o*stride - pad + k.
__device__ __forceinline__ bool strided_site(const int4 &c, int k, const Dims &d, int4 *o) {
  const int kz = k / (d.kh * d.kw), ky = (k / d.kw) % d.kh, kx = k % d.kw;
  int oz = c.y + d.pd - kz, oy = c.z + d.ph - ky, ox = c.w + d.pw - kx;
  if (oz < 0 || oy < 0 || ox < 0 || oz % d.sd || oy % d.sh || ox % d.sw) return false;
  oz /= d.sd;
  oy /= d.sh;
  ox /= d.sw;
  if (oz >= d.oD || oy >= d.oH || ox >= d.oW) return false;
  *o = make_int4(c.x, oz, oy, ox);
  return true;
}

// Input row under tap k of output site o's window, or -1.
__device__ __forceinline__ int window_row(const unsigned long long *__restrict__ tab, uint32_t mask, uint32_t shift,
                                          const int4 &o, int k, const Dims &d) {
  const int kz = k / (d.kh * d.kw), ky = (k / d.kw) % d.kh, kx = k % d.kw;
  const int iz = o.y * d.sd - d.pd + kz, iy = o.z * d.sh - d.ph + ky, ix = o.w * d.sw - d.pw + kx;
  if (iz < 0 || iz >= d.D || iy < 0 || iy >= d.H || ix < 0 || ix >= d.W) return -1;
  return lookup(tab, mask, shift, lin(o.x, iz, iy, ix, d.D, d.H, d.W));
}

// Strided conv: number the output sites in first-appearance order (input rows in row order, within a row the taps in
// tap order) in one pass.  The owner of a site is the smallest input row generating it; listed by (row, tap), the owners
// are the sites in first-appearance order.  Tiles of tile_rows input rows, taken by ticket, one thread per (row, tap):
//   A. every candidate site marks its table entry with the smallest generating row (atomicMin on kPending | row);
//   B. once every earlier tile has passed A (a look-back over zero aggregates), the entry holds the site's owner unless
//      a later tile's row generates it too, and those rows are larger: a candidate whose row the entry holds owns it;
//   C. the tile's owned sites get their ids from a block scan and a second decoupled look-back and are listed in id
//      order; one thread per site writes its coordinates and table entry (the id, or 0x7fffffff past out_cap), one
//      thread per (site, tap) its strided neighbour-map row.
// The grid is persistent: a block takes tickets until its tile starts past the last row, so no block waits on a tile
// that has not started.  desc: [0] the ticket, [1 + t] tile t's descriptor for B, [1 + tiles + t] for C, all zero before
// the launch.  s_own holds the tile's owned-tap masks (row r, tap k: bit k & 31 of word r * W + k / 32), s_off each
// row's first id within the tile, s_site the sites (r * K + k) of one chunk of ids.
constexpr int kSiteThreads = 256, kSiteMaskWords = 4096, kSiteMaxRows = 1024, kSiteList = 1024;
constexpr uint32_t kPending = 0x80000000u;

__device__ __forceinline__ uint32_t out_slot(const unsigned long long *tab, uint32_t mask, uint32_t shift, uint32_t key) {
  uint32_t h = hash32(key) >> shift;
  while (static_cast<uint32_t>(__ldcg(tab + h) >> 32) != key) h = (h + 1) & mask;
  return h;
}

__global__ void __launch_bounds__(kSiteThreads) rb_sites_kernel(
    const int32_t *__restrict__ coords, const int32_t *__restrict__ n_dev, long long n_cap, Dims d,
    const unsigned long long *__restrict__ tab_in, uint32_t mask_in, uint32_t shift_in, unsigned long long *tab_out,
    uint32_t mask_out, uint32_t shift_out, int32_t *__restrict__ out_coords, int32_t *__restrict__ n_out_dev,
    int out_cap, int32_t *__restrict__ nbr, unsigned long long *desc, int tiles, int tile_rows) {
  __shared__ uint32_t s_own[kSiteMaskWords];
  __shared__ int s_off[kSiteMaxRows];
  __shared__ int s_warp[kSiteThreads / 32];
  __shared__ unsigned int s_tile;
  __shared__ int s_prefix, s_total;
  __shared__ int s_site[kSiteList];
  const int K = d.kd * d.kh * d.kw, W = (K + 31) >> 5;
  const long long n = n_dev ? min(static_cast<long long>(n_dev[0]), n_cap) : n_cap;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  while (true) {
    __syncthreads();  // the previous tile's shared state is consumed
    if (threadIdx.x == 0) s_tile = static_cast<unsigned int>(atomicAdd(&desc[0], 1ull));
    __syncthreads();
    const unsigned int tile = s_tile;
    const long long tile0 = static_cast<long long>(tile) * tile_rows;
    if (tile0 >= n) return;  // past the last row: no later tile waits on this one
    const int rows = static_cast<int>(min(static_cast<long long>(tile_rows), n - tile0));
    for (int q = threadIdx.x; q < tile_rows * W; q += kSiteThreads) s_own[q] = 0u;
    // A: mark each candidate's site with the smallest generating row
    for (int q = threadIdx.x; q < rows * K; q += kSiteThreads) {
      const int r = q / K, k = q - r * K;
      const long long i = tile0 + r;
      const int4 c = *reinterpret_cast<const int4 *>(coords + static_cast<size_t>(i) * 4);
      if (c.x < 0 || c.x >= d.B || c.y < 0 || c.y >= d.D || c.z < 0 || c.z >= d.H || c.w < 0 || c.w >= d.W) continue;
      int4 o;
      if (!strided_site(c, k, d, &o)) continue;
      // a duplicate coordinate: the row the table holds (the later one) stands for it
      if (lookup(tab_in, mask_in, shift_in, lin(c.x, c.y, c.z, c.w, d.D, d.H, d.W)) != i) continue;
      const uint32_t key = lin(o.x, o.y, o.z, o.w, d.oD, d.oH, d.oW);
      const unsigned long long want = (static_cast<unsigned long long>(key) << 32) | kPending | static_cast<uint32_t>(i);
      uint32_t h = hash32(key) >> shift_out;
      for (uint32_t probes = 0;; ++probes) {
        if (probes > mask_out) {  // table full (far more sites than out_cap): flag it, the site is not numbered
          n_out_dev[3] = 1;
          break;
        }
        unsigned long long cur = __ldcg(tab_out + h);
        if (cur == kEmpty) {
          cur = atomicCAS(&tab_out[h], kEmpty, want);
          if (cur == kEmpty) break;
        }
        if (static_cast<uint32_t>(cur >> 32) == key) {
          atomicMin(&tab_out[h], want);
          break;
        }
        h = (h + 1) & mask_out;
      }
    }
    __threadfence();
    __syncthreads();
    if (wid == 0) lookback_exclusive_prefix(desc + 1, tile, 0);  // returns once every earlier tile has passed A
    __syncthreads();
    // B: a candidate owns its site when the entry still holds its row
    for (int q = threadIdx.x; q < rows * K; q += kSiteThreads) {
      const int r = q / K, k = q - r * K;
      const long long i = tile0 + r;
      const int4 c = *reinterpret_cast<const int4 *>(coords + static_cast<size_t>(i) * 4);
      if (c.x < 0 || c.x >= d.B || c.y < 0 || c.y >= d.D || c.z < 0 || c.z >= d.H || c.w < 0 || c.w >= d.W) continue;
      int4 o;
      if (!strided_site(c, k, d, &o)) continue;
      const uint32_t key = lin(o.x, o.y, o.z, o.w, d.oD, d.oH, d.oW);
      uint32_t h = hash32(key) >> shift_out;
      for (uint32_t probes = 0; probes <= mask_out; ++probes, h = (h + 1) & mask_out) {
        const unsigned long long e = __ldcg(tab_out + h);
        if (e == kEmpty) break;
        if (static_cast<uint32_t>(e >> 32) == key) {
          if (static_cast<uint32_t>(e) == (kPending | static_cast<uint32_t>(i))) atomicOr(&s_own[r * W + (k >> 5)], 1u << (k & 31));
          break;
        }
      }
    }
    __syncthreads();
    // C: ids in (row, tap) order: per-row offsets from a block scan, the tile's offset from the look-back
    const int rpt = (tile_rows + kSiteThreads - 1) / kSiteThreads, r0 = threadIdx.x * rpt;
    int cnt = 0;
    for (int r = r0; r < r0 + rpt && r < rows; ++r)
      for (int w = 0; w < W; ++w) cnt += __popc(s_own[r * W + w]);
    int inc = cnt;
  #pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, inc, s);
      if (lane >= s) inc += t;
    }
    if (lane == 31) s_warp[wid] = inc;
    __syncthreads();
    if (wid == 0) {
      const int v = lane < kSiteThreads / 32 ? s_warp[lane] : 0;
      int winc = v;
  #pragma unroll
      for (int s = 1; s < 32; s <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, winc, s);
        if (lane >= s) winc += t;
      }
      if (lane < kSiteThreads / 32) s_warp[lane] = winc - v;
      const int aggregate = __shfl_sync(0xffffffffu, winc, 31);
      const int prefix = lookback_exclusive_prefix(desc + 1 + tiles, tile, aggregate);
      if (lane == 0) {
        s_prefix = prefix;
        s_total = aggregate;
        if (tile0 + tile_rows >= n) n_out_dev[2] = prefix + aggregate;  // the last tile: raw count (clamped copy: [0])
      }
    }
    __syncthreads();
    int off = s_warp[wid] + inc - cnt;
    for (int r = r0; r < r0 + rpt && r < rows; ++r) {
      s_off[r] = off;
      for (int w = 0; w < W; ++w) off += __popc(s_own[r * W + w]);
    }
    const int prefix = s_prefix, total = s_total;
    for (int base = 0; base < total; base += kSiteList) {
      const int m = min(kSiteList, total - base);
      for (int r = r0; r < r0 + rpt && r < rows; ++r) {
        int j = s_off[r] - base;
        for (int w = 0; w < W && j < m; ++w)
          for (uint32_t bits = s_own[r * W + w]; bits && j < m; bits &= bits - 1u, ++j)
            if (j >= 0) s_site[j] = r * K + (w << 5) + __ffs(bits) - 1;
      }
      __syncthreads();
      for (int j = threadIdx.x; j < m; j += kSiteThreads) {
        const int r = s_site[j] / K, k = s_site[j] - r * K, id = prefix + base + j;
        int4 o;
        strided_site(*reinterpret_cast<const int4 *>(coords + static_cast<size_t>(tile0 + r) * 4), k, d, &o);
        const uint32_t key = lin(o.x, o.y, o.z, o.w, d.oD, d.oH, d.oW);
        // the entry now names the site's row of the OUTPUT index set: this table is that set's coordinate table
        atomicExch(&tab_out[out_slot(tab_out, mask_out, shift_out, key)],
                   (static_cast<unsigned long long>(key) << 32) | static_cast<uint32_t>(id < out_cap ? id : 0x7fffffff));
        if (id < out_cap) *reinterpret_cast<int4 *>(out_coords + static_cast<size_t>(id) * 4) = o;
      }
      for (int q = threadIdx.x; q < m * K; q += kSiteThreads) {
        const int j = q / K, k2 = q - j * K, id = prefix + base + j;
        if (id >= out_cap) break;  // ids grow with q
        const int r = s_site[j] / K, k = s_site[j] - r * K;
        const long long i = tile0 + r;
        int4 o;
        strided_site(*reinterpret_cast<const int4 *>(coords + static_cast<size_t>(i) * 4), k, d, &o);
        nbr[static_cast<size_t>(id) * K + k2] = k2 == k ? static_cast<int>(i) : window_row(tab_in, mask_in, shift_in, o, k2, d);
      }
      __syncthreads();
    }
  }
}

// One launch per resolution level after rb_sites: publishes the clamped output count / overflow flag and, when nbr_m
// is given, fills the 3-D SubM map of the level's residual blocks (rows of the output level, through tab_out, which
// rb_sites completed).
__global__ void __launch_bounds__(256) rb_level_neighbors_kernel(const int32_t *__restrict__ out_coords,
                                                                 int32_t *__restrict__ n_out_dev, long long out_cap,
                                                                 Dims dm, const unsigned long long *__restrict__ tab_out,
                                                                 uint32_t mask_out, uint32_t shift_out,
                                                                 int32_t *__restrict__ nbr_m) {
  const int raw = n_out_dev[2];
  const long long n = raw < out_cap ? raw : out_cap;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    n_out_dev[0] = static_cast<int32_t>(n);
    n_out_dev[1] = (raw > out_cap || n_out_dev[3]) ? 1 : 0;
  }
  if (!nbr_m) return;
  const int Km = dm.kd * dm.kh * dm.kw;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; q < n * Km; q += stride) {
    const int o = static_cast<int>(q / Km), k = static_cast<int>(q - static_cast<long long>(o) * Km);
    const int4 c = *reinterpret_cast<const int4 *>(out_coords + static_cast<size_t>(o) * 4);
    const int kz = k / (dm.kh * dm.kw), ky = (k / dm.kw) % dm.kh, kx = k % dm.kw;
    const int iz = c.y - dm.pd + kz, iy = c.z - dm.ph + ky, ix = c.w - dm.pw + kx;
    int r = -1;
    if (kz == dm.kd / 2 && ky == dm.kh / 2 && kx == dm.kw / 2) {
      r = o;
    } else if (iz >= 0 && iz < dm.D && iy >= 0 && iy < dm.H && ix >= 0 && ix < dm.W) {
      r = lookup(tab_out, mask_out, shift_out, lin(c.x, iz, iy, ix, dm.D, dm.H, dm.W));
    }
    nbr_m[q] = r;
  }
}

// ------------------------------------------------------------------ fp32 gather-GEMM
constexpr int TM = 64, TN = 64, KC = 16, LDA = TM + 4;

__global__ void __launch_bounds__(256) gather_gemm_fp32_kernel(const float *__restrict__ in,
                                                               const int32_t *__restrict__ nbr,
                                                               const int32_t *__restrict__ n_out_dev, long long n_cap,
                                                               int K, int Cin, int Cout,
                                                               const float *__restrict__ weight,
                                                               const float *__restrict__ scale,
                                                               const float *__restrict__ shift,
                                                               const float *__restrict__ residual, int relu,
                                                               float *__restrict__ out) {
  extern __shared__ int s_nbr[];                  // [TM][K]
  __shared__ __align__(16) float As[KC * LDA];   // [kc][row]
  __shared__ __align__(16) float Bs[KC * TN];    // [kc][col]
  const long long n = n_out_dev ? min(static_cast<long long>(n_out_dev[0]), n_cap) : n_cap;
  const long long row0 = static_cast<long long>(blockIdx.x) * TM;
  if (row0 >= n) return;
  const int col0 = blockIdx.y * TN;
  const int rows = static_cast<int>(min(static_cast<long long>(TM), n - row0));
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  for (int q = tid; q < TM * K; q += 256) s_nbr[q] = (q < rows * K) ? nbr[row0 * K + q] : -1;
  __syncthreads();
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const bool vecA = (Cin % 4 == 0);
  const int a_row = tid >> 2, a_seg = tid & 3;  // 64 rows x 4 segments of 4 channels
  for (int k = 0; k < K; ++k) {
    const int my = s_nbr[a_row * K + k];
    if (!__syncthreads_or(my >= 0)) continue;  // no row of this tile has tap k
    for (int c0 = 0; c0 < Cin; c0 += KC) {
      // gather A chunk
      float4 av = make_float4(0.f, 0.f, 0.f, 0.f);
      if (my >= 0) {
        const float *src = in + static_cast<size_t>(my) * Cin + c0 + a_seg * 4;
        if (vecA) {
          if (c0 + a_seg * 4 < Cin) av = __ldg(reinterpret_cast<const float4 *>(src));
        } else {
          const int left = Cin - (c0 + a_seg * 4);
          if (left > 0) av.x = __ldg(src);
          if (left > 1) av.y = __ldg(src + 1);
          if (left > 2) av.z = __ldg(src + 2);
          if (left > 3) av.w = __ldg(src + 3);
        }
      }
      As[(a_seg * 4 + 0) * LDA + a_row] = av.x;
      As[(a_seg * 4 + 1) * LDA + a_row] = av.y;
      As[(a_seg * 4 + 2) * LDA + a_row] = av.z;
      As[(a_seg * 4 + 3) * LDA + a_row] = av.w;
      // weight chunk W[k][c0 + r][col0 + c]
      for (int q = tid; q < KC * TN; q += 256) {
        const int r = q / TN, c = q - r * TN;
        float w = 0.f;
        if (c0 + r < Cin && col0 + c < Cout) w = __ldg(weight + (static_cast<size_t>(k) * Cin + c0 + r) * Cout + col0 + c);
        Bs[q] = w;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < KC; ++kk) {
        const float4 a = *reinterpret_cast<const float4 *>(&As[kk * LDA + ty * 4]);
        const float4 b = *reinterpret_cast<const float4 *>(&Bs[kk * TN + tx * 4]);
        const float ar[4] = {a.x, a.y, a.z, a.w}, br[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = ty * 4 + i;
    if (r >= rows) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = col0 + tx * 4 + j;
      if (c >= Cout) continue;
      float v = acc[i][j];
      if (scale) v = v * scale[c];
      if (shift) v = v + shift[c];
      if (residual) v = v + residual[(row0 + r) * Cout + c];
      if (relu) v = fmaxf(v, 0.f);
      out[(row0 + r) * Cout + c] = v;
    }
  }
}

// Unfused epilogue for API completeness (paddle.sparse.nn.BatchNorm / ReLU / sparse.add applied to an
// already materialised tensor): out = act(x * scale + shift (+ residual)).
__global__ void __launch_bounds__(256) rows_affine_act_kernel(const float *__restrict__ x,
                                                              const int32_t *__restrict__ n_dev, long long n_cap, int C,
                                                              const float *__restrict__ scale,
                                                              const float *__restrict__ shift,
                                                              const float *__restrict__ residual, int relu,
                                                              float *__restrict__ out) {
  const long long n = n_dev ? min(static_cast<long long>(n_dev[0]), n_cap) : n_cap;
  const long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (q >= n * C) return;
  const int c = static_cast<int>(q % C);
  float v = x[q];
  if (scale) v = v * scale[c];
  if (shift) v = v + shift[c];
  if (residual) v = v + residual[q];
  if (relu) v = fmaxf(v, 0.f);
  out[q] = v;
}

// Few input channels (the 5 -> 16 input layer, sparse_resnet.py:125-127): one thread per output row keeps all
// COUT accumulators in registers, weights of all taps live in shared memory; exact fp32 FMA chain.
template <int COUT>
__global__ void __launch_bounds__(128) small_cin_kernel(const float *__restrict__ in, const int32_t *__restrict__ nbr,
                                                        const int32_t *__restrict__ n_out_dev, long long n_cap, int K,
                                                        int Cin, const float *__restrict__ weight,
                                                        const float *__restrict__ scale, const float *__restrict__ shift,
                                                        const float *__restrict__ residual, int relu,
                                                        float *__restrict__ out, __half *__restrict__ out_h16,
                                                        int32_t *__restrict__ status) {
  // out_h16 (optional): the rows also (or only) as fp16 (hi, lo') pairs [n][hi COUT | lo' COUT] for the fp16-pair
  // tensor-core layers that follow (csrc/sparse_conv_f16.cu): saves the separate conversion pass
  extern __shared__ float s_w[];  // [K][Cin][COUT]
  const long long n = n_out_dev ? min(static_cast<long long>(n_out_dev[0]), n_cap) : n_cap;
  if (static_cast<long long>(blockIdx.x) * blockDim.x >= n) return;
  for (int q = threadIdx.x; q < K * Cin * COUT; q += blockDim.x) s_w[q] = weight[q];
  __syncthreads();
  const long long row = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (row >= n) return;
  float acc[COUT];
#pragma unroll
  for (int c = 0; c < COUT; ++c) acc[c] = 0.f;
  const int32_t *nb = nbr + row * K;
  // Taps in batches of kTapBatch: first all neighbour indices of the batch, then all their (<= 8-channel) rows, then
  // the FMAs - two memory latencies per batch instead of two per tap.  The FMA order (tap, then channel) and the
  // skipping of missing neighbours are those of the plain loop, so results are bit-identical to it.
  constexpr int kTapBatch = 9, kMaxCin = 8;
  for (int k0 = 0; k0 < K; k0 += kTapBatch) {
    int src[kTapBatch];
#pragma unroll
    for (int j = 0; j < kTapBatch; ++j) src[j] = (k0 + j < K) ? __ldg(nb + k0 + j) : -1;
    float xv[kTapBatch][kMaxCin];
#pragma unroll
    for (int j = 0; j < kTapBatch; ++j) {
      const float *x = in + static_cast<size_t>(src[j] < 0 ? 0 : src[j]) * Cin;
#pragma unroll
      for (int ci = 0; ci < kMaxCin; ++ci) xv[j][ci] = (src[j] >= 0 && ci < Cin) ? __ldg(x + ci) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < kTapBatch; ++j) {
      if (src[j] < 0) continue;
      const float *w = s_w + (k0 + j) * Cin * COUT;
#pragma unroll
      for (int ci = 0; ci < kMaxCin; ++ci) {
        if (ci < Cin) {
#pragma unroll
          for (int c = 0; c < COUT; ++c) acc[c] = fmaf(xv[j][ci], w[ci * COUT + c], acc[c]);
        }
      }
    }
  }
  bool ovf = false;
#pragma unroll
  for (int c = 0; c < COUT; ++c) {
    float v = acc[c];
    if (scale) v = v * scale[c];
    if (shift) v = v + shift[c];
    if (residual) v = v + residual[row * COUT + c];
    if (relu) v = fmaxf(v, 0.f);
    acc[c] = v;
  }
  if (out) {
    float4 *o = reinterpret_cast<float4 *>(out + row * COUT);
#pragma unroll
    for (int c = 0; c < COUT; c += 4) o[c / 4] = make_float4(acc[c], acc[c + 1], acc[c + 2], acc[c + 3]);
  }
  if (out_h16) {
    uint32_t hw[COUT / 2], lw[COUT / 2];
#pragma unroll
    for (int c = 0; c < COUT; c += 2) {
      __half h0, l0, h1, l1;
      split_h16(acc[c], h0, l0, ovf);
      split_h16(acc[c + 1], h1, l1, ovf);
      const __half2 hh = __halves2half2(h0, h1), ll = __halves2half2(l0, l1);
      hw[c / 2] = *reinterpret_cast<const uint32_t *>(&hh);
      lw[c / 2] = *reinterpret_cast<const uint32_t *>(&ll);
    }
    uint4 *o = reinterpret_cast<uint4 *>(out_h16 + row * 2 * COUT);  // [hi COUT | lo' COUT] (COUT = 16 or 32: one group)
#pragma unroll
    for (int q = 0; q < COUT / 8; ++q) o[q] = make_uint4(hw[4 * q], hw[4 * q + 1], hw[4 * q + 2], hw[4 * q + 3]);
#pragma unroll
    for (int q = 0; q < COUT / 8; ++q) o[COUT / 8 + q] = make_uint4(lw[4 * q], lw[4 * q + 1], lw[4 * q + 2], lw[4 * q + 3]);
    if (ovf && status) atomicOr(status, 1);
  }
}

unsigned int persistent_grid(long long work_items) {
  const long long need = (work_items + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 8;  // 8 CTAs of 256 threads per SM = full occupancy
  return static_cast<unsigned int>(need < cap ? (need > 0 ? need : 1) : cap);
}

int make_dims(int batch, const int *sp, const int *ks, const int *st, const int *pd, int subm, Dims *d) {
  if (!sp || !ks || batch < 1) return P3D_ERR_INVALID_ARG;
  d->B = batch;
  d->D = sp[0];
  d->H = sp[1];
  d->W = sp[2];
  d->kd = ks[0];
  d->kh = ks[1];
  d->kw = ks[2];
  if (d->D < 1 || d->H < 1 || d->W < 1 || d->kd < 1 || d->kh < 1 || d->kw < 1) return P3D_ERR_INVALID_ARG;
  if (subm) {
    if (!(d->kd & 1) || !(d->kh & 1) || !(d->kw & 1)) return P3D_ERR_UNSUPPORTED;
    d->sd = d->sh = d->sw = 1;
    d->pd = d->kd / 2;
    d->ph = d->kh / 2;
    d->pw = d->kw / 2;
    d->oD = d->D;
    d->oH = d->H;
    d->oW = d->W;
  } else {
    if (!st || !pd) return P3D_ERR_INVALID_ARG;
    d->sd = st[0];
    d->sh = st[1];
    d->sw = st[2];
    d->pd = pd[0];
    d->ph = pd[1];
    d->pw = pd[2];
    if (d->sd < 1 || d->sh < 1 || d->sw < 1 || d->pd < 0 || d->ph < 0 || d->pw < 0) return P3D_ERR_INVALID_ARG;
    d->oD = (d->D + 2 * d->pd - d->kd) / d->sd + 1;
    d->oH = (d->H + 2 * d->ph - d->kh) / d->sh + 1;
    d->oW = (d->W + 2 * d->pw - d->kw) / d->sw + 1;
    if (d->oD < 1 || d->oH < 1 || d->oW < 1) return P3D_ERR_INVALID_ARG;
  }
  if (static_cast<long long>(batch) * d->D * d->H * d->W >= 0xffffffffll) return P3D_ERR_UNSUPPORTED;
  if (d->kd * d->kh * d->kw > 125) return P3D_ERR_UNSUPPORTED;
  return P3D_OK;
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_sparse_conv_gather_gemm_fp32(const float *in, const int32_t *nbr, const int32_t *n_out_dev,
                                                int64_t n_out_cap, int K, int Cin, int Cout, const float *weight,
                                                const float *scale, const float *shift, const float *residual,
                                                int relu, float *out, p3d_stream_t stream) {
  if (n_out_cap < 0 || K < 1 || Cin < 1 || Cout < 1 || !weight || (n_out_cap && (!in || !nbr || !out)))
    return P3D_ERR_INVALID_ARG;
  if (n_out_cap == 0) return P3D_OK;
  if ((Cin % 4 == 0) && (reinterpret_cast<uintptr_t>(in) & 15)) return P3D_ERR_INVALID_ARG;
  if (Cin <= 8 && (Cout == 16 || Cout == 32) && static_cast<size_t>(K) * Cin * Cout * 4 <= 40 * 1024) {
    const size_t sw = static_cast<size_t>(K) * Cin * Cout * sizeof(float);
    if (Cout == 16)
      small_cin_kernel<16><<<div_up(n_out_cap, 128), 128, sw, static_cast<cudaStream_t>(stream)>>>(
          in, nbr, n_out_dev, n_out_cap, K, Cin, weight, scale, shift, residual, relu, out, nullptr, nullptr);
    else
      small_cin_kernel<32><<<div_up(n_out_cap, 128), 128, sw, static_cast<cudaStream_t>(stream)>>>(
          in, nbr, n_out_dev, n_out_cap, K, Cin, weight, scale, shift, residual, relu, out, nullptr, nullptr);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
  }
  const size_t smem = static_cast<size_t>(TM) * K * sizeof(int);
  if (smem > 40 * 1024) return P3D_ERR_UNSUPPORTED;
  dim3 grid(div_up(n_out_cap, TM), div_up(Cout, TN));
  gather_gemm_fp32_kernel<<<grid, 256, smem, static_cast<cudaStream_t>(stream)>>>(
      in, nbr, n_out_dev, n_out_cap, K, Cin, Cout, weight, scale, shift, residual, relu, out);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

// The few-input-channel layer (5 -> 16 input conv) with fp16-pair output rows for the tensor-core layers behind it:
// out_f32 and / or out_h16 ([n][hi Cout | lo' Cout] halfs) may be given; exact fp32 FMA chain as p3d_sparse_conv_gather_gemm.
extern "C" int p3d_sparse_conv_small_cin_h16(const float *in, const int32_t *nbr, const int32_t *n_out_dev, int64_t n_out_cap,
                                             int K, int Cin, int Cout, const float *weight, const float *scale,
                                             const float *shift, int relu, float *out_f32, void *out_h16,
                                             int32_t *status_dev, p3d_stream_t stream) {
  if (n_out_cap < 0 || K < 1 || !weight || (!out_f32 && !out_h16) || (n_out_cap && (!in || !nbr))) return P3D_ERR_INVALID_ARG;
  if (n_out_cap == 0) return P3D_OK;
  if (!(Cin <= 8 && (Cout == 16 || Cout == 32) && static_cast<size_t>(K) * Cin * Cout * 4 <= 40 * 1024)) return P3D_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(out_f32) & 15) || (reinterpret_cast<uintptr_t>(out_h16) & 15)) return P3D_ERR_INVALID_ARG;
  const size_t sw = static_cast<size_t>(K) * Cin * Cout * sizeof(float);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (Cout == 16)
    small_cin_kernel<16><<<div_up(n_out_cap, 128), 128, sw, st>>>(in, nbr, n_out_dev, n_out_cap, K, Cin, weight, scale, shift, nullptr,
                                                                  relu, out_f32, static_cast<__half *>(out_h16), status_dev);
  else
    small_cin_kernel<32><<<div_up(n_out_cap, 128), 128, sw, st>>>(in, nbr, n_out_dev, n_out_cap, K, Cin, weight, scale, shift, nullptr,
                                                                  relu, out_f32, static_cast<__half *>(out_h16), status_dev);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" int p3d_sparse_affine_act(const float *x, const int32_t *n_dev, int64_t n_cap, int C, const float *scale,
                                     const float *shift, const float *residual, int relu, float *out,
                                     p3d_stream_t stream) {
  if (n_cap < 0 || C < 1 || (n_cap && (!x || !out))) return P3D_ERR_INVALID_ARG;
  if (n_cap == 0) return P3D_OK;
  rows_affine_act_kernel<<<div_up(n_cap * C, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, n_dev, n_cap, C, scale, shift, residual, relu, out);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

// ------------------------------------------------------------------ coordinate tables
// One table per index set (resolution level).  The level-0 table is built from the voxel coordinates; the table of a
// strided conv's OUTPUT set is a by-product of enumerating its sites, and is what the next stage's SubM rulebook and
// the next strided conv look coordinates up in — so every level's table is built exactly once per frame.  The
// scratch-workspace entry points run the same code on tables carved out of their workspace.
namespace {
// A table of rows_cap rows: `cap` 64-bit entries (2x the rows, a power of two), then the site numbering's scratch of a
// strided conv writing into it: a ticket and `tiles` look-back descriptors (two per input tile), at least one per 64
// entries and never fewer than kMinTiles, so that a tile's rows and owned-tap masks fit rb_sites' shared memory for any
// input capacity check_level accepts (2^24 rows, 125 taps: 1024 rows of 4 mask words).
constexpr uint32_t kMinTiles = 32768;
struct Tab {
  unsigned long long *p;
  uint32_t cap, shift, tiles;
  unsigned long long *scratch() const { return p + cap; }
};
uint32_t tab_cap(int64_t rows_cap) { return next_pow2(static_cast<uint64_t>(rows_cap > 512 ? rows_cap : 512) * 2); }
uint32_t tab_tiles(uint32_t cap) { return cap / 64 > kMinTiles ? cap / 64 : kMinTiles; }

size_t tab_bytes(int64_t rows_cap) {
  const uint32_t cap = tab_cap(rows_cap);
  return align_up((static_cast<size_t>(cap) + 1 + tab_tiles(cap)) * 8);
}

bool tab_of(void *mem, size_t bytes, int64_t rows_cap, Tab *t) {
  if (rows_cap > kMaxRows) return false;
  t->cap = tab_cap(rows_cap);
  t->tiles = tab_tiles(t->cap);
  t->shift = 32;
  for (uint32_t x = t->cap; x > 1; x >>= 1) --t->shift;
  t->p = static_cast<unsigned long long *>(mem);
  return mem && bytes >= tab_bytes(rows_cap) && !(reinterpret_cast<uintptr_t>(mem) & 15);
}

// The tables of p3d_sparse_rulebook_workspace_bytes(n_in_cap, n_out_cap): input set first, then output set.
int carve_tables(void *ws, size_t ws_bytes, int64_t n_in_cap, int64_t n_out_cap, Tab *ti, Tab *to) {
  const size_t in_bytes = tab_bytes(n_in_cap), out_bytes = tab_bytes(n_out_cap);
  if (ws_bytes < in_bytes + out_bytes) return P3D_ERR_WORKSPACE;
  char *p = static_cast<char *>(ws);
  return tab_of(p, in_bytes, n_in_cap, ti) && tab_of(p + in_bytes, out_bytes, n_out_cap, to) ? P3D_OK
                                                                                             : P3D_ERR_INVALID_ARG;
}

// Argument checks of the SubM / strided entry points; bad_buffers = the caller's own table or workspace check.
int check_subm(const int32_t *coords, int64_t n_cap, int batch, const int *spatial_host, const int *ksize_host,
               const int32_t *nbr, bool bad_buffers, Dims *d) {
  int rc = make_dims(batch, spatial_host, ksize_host, nullptr, nullptr, 1, d);
  if (rc) return rc;
  if (n_cap < 0 || n_cap > 0x7fffffff / 128 || bad_buffers || (n_cap && (!coords || !nbr)) ||
      (reinterpret_cast<uintptr_t>(coords) & 15))
    return P3D_ERR_INVALID_ARG;
  return P3D_OK;
}

int check_level(const int32_t *coords, int64_t n_in_cap, int batch, const int *spatial_host, const int *ksize_host,
                const int *stride_host, const int *pad_host, const int32_t *out_coords, const int32_t *n_out_dev,
                int64_t out_cap, const int32_t *nbr, bool bad_buffers, Dims *d) {
  int rc = make_dims(batch, spatial_host, ksize_host, stride_host, pad_host, 0, d);
  if (rc) return rc;
  if (n_in_cap < 0 || out_cap < 1 || n_in_cap > 0x7fffffff / 128 || out_cap > 0x7fffffff / 128 || bad_buffers ||
      !n_out_dev || !out_coords || !nbr || (n_in_cap && !coords))
    return P3D_ERR_INVALID_ARG;
  if ((reinterpret_cast<uintptr_t>(coords) & 15) || (reinterpret_cast<uintptr_t>(out_coords) & 15))
    return P3D_ERR_INVALID_ARG;
  if (static_cast<long long>(batch) * d->oD * d->oH * d->oW >= 0xffffffffll) return P3D_ERR_UNSUPPORTED;
  return P3D_OK;
}

int build_table(const int32_t *coords, const int32_t *n_dev, int64_t n_cap, const Dims &d, const Tab &t,
                cudaStream_t st) {
  P3D_CUDA_CHECK(cudaMemsetAsync(t.p, 0xff, static_cast<size_t>(t.cap) * 8, st));
  if (n_cap > 0) {
    rb_insert_kernel<<<div_up(n_cap, 256), 256, 0, st>>>(coords, n_dev, static_cast<int>(n_cap), d, t.p, t.cap - 1, t.shift);
    P3D_LAUNCH_CHECK();
  }
  return P3D_OK;
}

int subm_map(const int32_t *coords, const int32_t *n_dev, int64_t n_cap, const Dims &d, const Tab &t, int32_t *nbr,
             cudaStream_t st) {
  const int K = d.kd * d.kh * d.kw;
  rb_neighbors_kernel<<<persistent_grid(n_cap * K), 256, 0, st>>>(coords, n_dev, n_cap, d, t.p, t.cap - 1, t.shift, nbr);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

// One resolution level in two launches: output sites + table `to` of the strided conv d (inputs looked up in `ti`) with
// its neighbour map, then the counters and, when nbr_subm is given, the SubM map dm of the new level.
int level_maps(const int32_t *coords, const int32_t *n_in_dev, int64_t n_in_cap, const Dims &d, const Tab &ti,
               int32_t *out_coords, int32_t *n_out_dev, int64_t out_cap, const Tab &to, int32_t *nbr, const Dims &dm,
               int32_t *nbr_subm, cudaStream_t st) {
  const int Km = nbr_subm ? dm.kd * dm.kh * dm.kw : 0;
  P3D_CUDA_CHECK(cudaMemsetAsync(to.p, 0xff, static_cast<size_t>(to.cap) * 8, st));
  P3D_CUDA_CHECK(cudaMemsetAsync(n_out_dev, 0, sizeof(int32_t) * 4, st));
  if (n_in_cap > 0) {
    // 32 input rows per tile (one thread per (row, tap)), wider when the tiles would not fit the scratch
    const int words = (d.kd * d.kh * d.kw + 31) / 32;
    const long long half = to.tiles / 2;
    int rows = static_cast<int>(((n_in_cap + half - 1) / half + 31) / 32 * 32);
    if (rows < 32) rows = 32;
    if (rows > kSiteMaxRows || rows * words > kSiteMaskWords) return P3D_ERR_UNSUPPORTED;
    const unsigned int tiles = div_up(n_in_cap, rows);
    P3D_CUDA_CHECK(cudaMemsetAsync(to.scratch(), 0, (2 * static_cast<size_t>(tiles) + 1) * 8, st));
    const unsigned int grid = std::min(tiles, static_cast<unsigned int>(num_sms()) * 8);
    rb_sites_kernel<<<grid, kSiteThreads, 0, st>>>(coords, n_in_dev, n_in_cap, d, ti.p, ti.cap - 1, ti.shift, to.p,
                                                    to.cap - 1, to.shift, out_coords, n_out_dev,
                                                    static_cast<int>(out_cap), nbr, to.scratch(),
                                                    static_cast<int>(tiles), rows);
    P3D_LAUNCH_CHECK();
  }
  rb_level_neighbors_kernel<<<persistent_grid(out_cap * Km), 256, 0, st>>>(out_coords, n_out_dev, out_cap, dm, to.p,
                                                                          to.cap - 1, to.shift, nbr_subm);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
}  // namespace

extern "C" size_t p3d_sparse_table_bytes(int64_t rows_cap) {
  if (rows_cap < 0 || rows_cap > kMaxRows) return 0;
  return tab_bytes(rows_cap);
}

extern "C" int p3d_sparse_table_build(const int32_t *coords, const int32_t *n_dev, int64_t n_cap, int batch,
                                      const int *spatial_host, void *table, size_t table_bytes, p3d_stream_t stream) {
  const int one[3] = {1, 1, 1};
  Dims d;
  int rc = make_dims(batch, spatial_host, one, nullptr, nullptr, 1, &d);
  if (rc) return rc;
  Tab t;
  if (n_cap < 0 || n_cap > 0x7fffffff / 128 || !tab_of(table, table_bytes, n_cap, &t) || (n_cap && !coords) ||
      (reinterpret_cast<uintptr_t>(coords) & 15))
    return P3D_ERR_INVALID_ARG;
  return build_table(coords, n_dev, n_cap, d, t, static_cast<cudaStream_t>(stream));
}

extern "C" int p3d_sparse_rulebook_subm_t(const int32_t *coords, const int32_t *n_dev, int64_t n_cap, int batch,
                                          const int *spatial_host, const int *ksize_host, const void *table,
                                          size_t table_bytes, int32_t *nbr, p3d_stream_t stream) {
  Dims d;
  Tab t;
  const bool bad = !tab_of(const_cast<void *>(table), table_bytes, n_cap, &t);
  const int rc = check_subm(coords, n_cap, batch, spatial_host, ksize_host, nbr, bad, &d);
  if (rc || n_cap == 0) return rc;
  return subm_map(coords, n_dev, n_cap, d, t, nbr, static_cast<cudaStream_t>(stream));
}

extern "C" int p3d_sparse_rulebook_level_t(const int32_t *coords, const int32_t *n_in_dev, int64_t n_in_cap, int batch,
                                           const int *spatial_host, const int *ksize_host, const int *stride_host,
                                           const int *pad_host, const void *table_in, size_t table_in_bytes,
                                           int32_t *out_coords, int32_t *n_out_dev, int64_t out_cap, void *table_out,
                                           size_t table_out_bytes, int32_t *nbr, const int *subm_ksize_host,
                                           int32_t *nbr_subm, p3d_stream_t stream) {
  Dims d;
  Tab ti, to;
  const bool bad = !tab_of(const_cast<void *>(table_in), table_in_bytes, n_in_cap, &ti) ||
                   !tab_of(table_out, table_out_bytes, out_cap, &to) || (nbr_subm && !subm_ksize_host);
  int rc = check_level(coords, n_in_cap, batch, spatial_host, ksize_host, stride_host, pad_host, out_coords, n_out_dev,
                       out_cap, nbr, bad, &d);
  if (rc) return rc;
  Dims dm = d;
  if (nbr_subm) {
    const int osp[3] = {d.oD, d.oH, d.oW};
    rc = make_dims(batch, osp, subm_ksize_host, nullptr, nullptr, 1, &dm);
    if (rc) return rc;
  }
  return level_maps(coords, n_in_dev, n_in_cap, d, ti, out_coords, n_out_dev, out_cap, to, nbr, dm, nbr_subm,
                    static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------ scratch-workspace entry points (the Paddle ops)
extern "C" size_t p3d_sparse_rulebook_workspace_bytes(int64_t n_in_cap, int64_t n_out_cap) {
  if (n_in_cap < 0 || n_out_cap < 0 || n_in_cap > kMaxRows || n_out_cap > kMaxRows) return 0;
  return tab_bytes(n_in_cap) + tab_bytes(n_out_cap);
}

extern "C" int p3d_sparse_rulebook_subm(const int32_t *coords, const int32_t *n_in_dev, int64_t n_in_cap, int batch,
                                        const int *spatial_host, const int *ksize_host, int32_t *nbr,
                                        void *workspace, size_t workspace_bytes, p3d_stream_t stream) {
  Dims d;
  Tab t, unused;
  int rc = check_subm(coords, n_in_cap, batch, spatial_host, ksize_host, nbr, !workspace, &d);
  if (rc || n_in_cap == 0) return rc;
  if ((rc = carve_tables(workspace, workspace_bytes, n_in_cap, 0, &t, &unused))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if ((rc = build_table(coords, n_in_dev, n_in_cap, d, t, st))) return rc;
  return subm_map(coords, n_in_dev, n_in_cap, d, t, nbr, st);
}

extern "C" int p3d_sparse_rulebook_conv(const int32_t *coords, const int32_t *n_in_dev, int64_t n_in_cap, int batch,
                                        const int *spatial_host, const int *ksize_host, const int *stride_host,
                                        const int *pad_host, int32_t *out_coords, int32_t *n_out_dev,
                                        int64_t out_cap, int32_t *nbr, void *workspace, size_t workspace_bytes,
                                        p3d_stream_t stream) {
  Dims d;
  Tab ti, to;
  int rc = check_level(coords, n_in_cap, batch, spatial_host, ksize_host, stride_host, pad_host, out_coords, n_out_dev,
                       out_cap, nbr, !workspace, &d);
  if (rc || (rc = carve_tables(workspace, workspace_bytes, n_in_cap, out_cap, &ti, &to))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if ((rc = build_table(coords, n_in_dev, n_in_cap, d, ti, st))) return rc;
  return level_maps(coords, n_in_dev, n_in_cap, d, ti, out_coords, n_out_dev, out_cap, to, nbr, d, nullptr, st);
}
