// hard_voxelize for sm_90a — deterministic, CPU-semantics exact.
//
// Replaces the reference's 7-kernel + cumsum pipeline over three dense 332 MB grids
// (paddle3d/ops/voxel/voxelize_op.cu:208-346) with a hash of the occupied cells only:
//
//   K0 vox_init        table <- EMPTY, scan descriptors / voxel counts <- 0, overflow lists <- INF   (one launch)
//   K1 vox_insert      per point: cell id, open-addressing insert; the 64-bit entry is
//                      (cell << 32 | point index) and is reduced with one atomicMin, so each
//                      occupied cell ends up holding its FIRST point — the quantity the CPU
//                      kernel's first-appearance numbering is built on (voxelize_op.cc:59-69).
//                      Same-cell lanes of a warp are aggregated with __match_any_sync: only the
//                      lowest lane (smallest index) touches the table.
//   K2 vox_rank        single-pass decoupled-look-back scan over "is first point of its cell"
//                      flags -> voxel id (rank < max_voxels, else dropped: .cc:61-64), coords.
//   K3 vox_slots       per point: arrival number inside its voxel (one atomicAdd); the first C arrivals are recorded
//                      as they come, later ones (voxels with more than C = max(4P, 32) points; for P > 16 every point takes this path, see cand_slots) keep their P smallest
//                      indices with a cascade of atomicMin (deterministic under any interleaving: slot s always
//                      converges to the (s+1)-th smallest index).
//   K3b vox_select     per (voxel, slot): the P smallest recorded indices in ascending order - the CPU kernel's
//                      "first P points in input order" (.cc:71-79) - by rank counting (indices are distinct).
//   K4 vox_write       gather-formulated single pass over the outputs: every float4 of
//                      voxels[max_voxels, P, F] is written exactly once (point value or zero),
//                      coalesced, plus num_points_per_voxel and the zero tail of coords.
//                      This is the HBM-roofline kernel: 4NF + 4VPF + 12V + 4V algorithmic bytes.
//
// All intermediate state (8*cap + 4*(N + cap + V*(2P + C + 1)) bytes, of which only the rows of live voxels are touched)
// is L2-resident on an H100 (50 MB L2).
#include <limits.h>

#include "common.cuh"

namespace p3d {
namespace {

constexpr unsigned long long kEmpty = ~0ull;
constexpr int kInf = 0x7fffffff;
constexpr int kScanBlock = 512;
constexpr int kScanItems = 4;                       // consecutive points per thread of the rank scan
constexpr int kScanTile = kScanBlock * kScanItems;  // points per block: 147 blocks at 300k points (one per SM), <= 5 look-back rounds

struct VoxGeom {
  float min_x, min_y, min_z;
  float vs_x, vs_y, vs_z;
  int gx, gy, gz;
};

struct VoxWs {
  unsigned long long *table;   // [cap] (cell << 32 | first point index)
  unsigned long long *desc;    // [nblocks + 1]  desc[0] = ticket, desc[1 + b] = (status << 32 | value)
  int32_t *pt_slot;            // [N] table slot of each point, -1 = outside the grid
  int32_t *slot_vox;           // [cap] voxel id of an occupied slot (-1 = beyond max_voxels)
  int32_t *lists;              // [V, P] the P smallest point indices of each voxel, ascending (written by K3b)
  int32_t *count;              // [V] points of each voxel (zeroed by K0)
  int32_t *cand;               // [V, C] point indices in ARRIVAL order, the first C arrivals of each voxel (K3)
  int32_t *ovf;                // [V, P] P smallest indices among the arrivals beyond C (atomicMin cascade), INF-filled by K0
  int C;                       // candidate slots per voxel
  uint32_t cap, shift;
  unsigned int nblocks;
  size_t bytes;
};

// Candidate slots per voxel: a voxel's first C points (in arrival order) are kept as they come, one atomicAdd each;
// only voxels with more than C points fall back to the atomicMin cascade for the rest.
inline int cand_slots(int P) {
  // Recording arrivals costs one same-address atomicAdd per point of a voxel and the selection is quadratic in the
  // voxel's population; it pays off for the small P of the voxel models (C3, P = 10) and not for pillar models (C2,
  // P = 32, pillars of 200 points).  C = 0 selects the all-cascade path: K3 cascades every point into `ovf`, which K4 reads directly.
  if (P > 16) return 0;
  int c = 4 * P > 32 ? 4 * P : 32;
  return (c + 3) & ~3;
}

VoxWs carve(void *ws, int64_t n, int P, int V) {
  VoxWs w;
  Carver c(ws);
  w.cap = next_pow2(static_cast<uint64_t>(n > 512 ? n : 512) * 2);
  w.shift = 32;
  for (uint32_t x = w.cap; x > 1; x >>= 1) --w.shift;
  w.nblocks = div_up(n > 0 ? n : 1, kScanTile);
  w.table = c.take<unsigned long long>(w.cap);
  w.desc = c.take<unsigned long long>(w.nblocks + 1);
  w.pt_slot = c.take<int32_t>(n > 0 ? n : 1);
  w.slot_vox = c.take<int32_t>(w.cap);
  w.C = cand_slots(P);
  w.count = c.take<int32_t>(static_cast<size_t>(V));
  w.cand = c.take<int32_t>(static_cast<size_t>(V) * (w.C > 0 ? w.C : 1));
  w.ovf = c.take<int32_t>(static_cast<size_t>(V) * P);
  w.lists = w.C > 0 ? c.take<int32_t>(static_cast<size_t>(V) * P) : w.ovf;  // all-cascade path: the cascade's lists are final
  w.bytes = c.off;
  return w;
}

// ---------------------------------------------------------------- K0
__global__ void vox_init_kernel(uint4 *table16, size_t n_table16, uint4 *desc16, size_t n_desc16, uint4 *lists16,
                                size_t n_lists16, uint4 *count16, size_t n_count16) {
  pdl_trigger();
  pdl_wait();
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint4 ones = make_uint4(~0u, ~0u, ~0u, ~0u);
  const uint4 zero = make_uint4(0, 0, 0, 0);
  const uint4 inf = make_uint4(kInf, kInf, kInf, kInf);
  for (size_t i = tid; i < n_table16; i += stride) table16[i] = ones;
  for (size_t i = tid; i < n_desc16; i += stride) desc16[i] = zero;
  for (size_t i = tid; i < n_lists16; i += stride) lists16[i] = inf;
  for (size_t i = tid; i < n_count16; i += stride) count16[i] = zero;
}

// ---------------------------------------------------------------- K1
__device__ __forceinline__ int cell_of(const float *__restrict__ pt, const VoxGeom &g) {
  // fp32 subtract, IEEE fp32 divide, floor — exactly voxelize_op.cc:37-45
  const float fx = floorf(__fdiv_rn(__fsub_rn(pt[0], g.min_x), g.vs_x));
  const float fy = floorf(__fdiv_rn(__fsub_rn(pt[1], g.min_y), g.vs_y));
  const float fz = floorf(__fdiv_rn(__fsub_rn(pt[2], g.min_z), g.vs_z));
  // The reference CPU kernel converts with an x86 cvttss2si: NaN (and anything outside int range) becomes
  // INT_MIN and is dropped by the `< 0` test.  CUDA's float->int turns NaN into 0, so reject it explicitly.
  if (!(fx == fx) || !(fy == fy) || !(fz == fz)) return -1;
  const int cx = static_cast<int>(fx), cy = static_cast<int>(fy), cz = static_cast<int>(fz);
  if (cx < 0 || cx >= g.gx || cy < 0 || cy >= g.gy || cz < 0 || cz >= g.gz) return -1;
  return (cz * g.gy + cy) * g.gx + cx;
}

__global__ void __launch_bounds__(256) vox_insert_kernel(const float *__restrict__ points, int n, int F, VoxGeom g,
                                                         unsigned long long *__restrict__ table, uint32_t mask,
                                                         uint32_t shift, int32_t *__restrict__ pt_slot) {
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned active = __ballot_sync(0xffffffffu, i < n);
  if (i >= n) return;
  const int cell = cell_of(points + static_cast<size_t>(i) * F, g);
  // warp aggregation: lanes that fall in the same cell elect their lowest lane (= smallest index)
  const unsigned peers = __match_any_sync(active, cell);
  const int leader = __ffs(peers) - 1;
  const int lane = threadIdx.x & 31;
  int slot = -1;
  if (cell >= 0 && lane == leader) {
    const unsigned long long want = (static_cast<unsigned long long>(cell) << 32) | static_cast<uint32_t>(i);
    uint32_t h = hash32(static_cast<uint32_t>(cell)) >> shift;
    while (true) {
      unsigned long long cur = table[h];
      if (cur == kEmpty) {
        cur = atomicCAS(&table[h], kEmpty, want);
        if (cur == kEmpty) break;
      }
      if (static_cast<uint32_t>(cur >> 32) == static_cast<uint32_t>(cell)) {
        if (want < cur) atomicMin(&table[h], want);
        break;
      }
      h = (h + 1) & mask;
    }
    slot = static_cast<int>(h);
  }
  slot = __shfl_sync(peers, slot, leader);
  pt_slot[i] = slot;
}

// ---------------------------------------------------------------- K2
__global__ void __launch_bounds__(kScanBlock) vox_rank_kernel(const unsigned long long *__restrict__ table,
                                                              const int32_t *__restrict__ pt_slot, int n,
                                                              int max_voxels, VoxGeom g,
                                                              unsigned long long *__restrict__ desc,
                                                              int32_t *__restrict__ slot_vox,
                                                              int32_t *__restrict__ coords, int coord_stride,
                                                              int coord_off, int batch_id,
                                                              int32_t *__restrict__ num_voxels) {
  pdl_trigger();
  pdl_wait();
  __shared__ unsigned int s_bid;
  __shared__ int s_warp[kScanBlock / 32];
  __shared__ int s_prefix;
  if (threadIdx.x == 0) s_bid = static_cast<unsigned int>(atomicAdd(&desc[0], 1ull));
  __syncthreads();
  const unsigned int bid = s_bid;
  const int i0 = static_cast<int>(bid) * kScanTile + threadIdx.x * kScanItems;
  int slot[kScanItems];
  unsigned long long entry[kScanItems];
  if (i0 + kScanItems <= n) {
    const int4 v4 = *reinterpret_cast<const int4 *>(pt_slot + i0);  // i0 is a multiple of 4, pt_slot 256-byte aligned
    slot[0] = v4.x;
    slot[1] = v4.y;
    slot[2] = v4.z;
    slot[3] = v4.w;
  } else {
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) slot[k] = (i0 + k < n) ? pt_slot[i0 + k] : -1;
  }
  static_assert(kScanItems == 4, "the vector load above is written for 4 items per thread");
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) entry[k] = slot[k] >= 0 ? table[slot[k]] : 0ull;
  unsigned int flags = 0u;  // bit k: point i0 + k is the first point of its cell
#pragma unroll
  for (int k = 0; k < kScanItems; ++k)
    if (slot[k] >= 0 && static_cast<uint32_t>(entry[k]) == static_cast<uint32_t>(i0 + k)) flags |= 1u << k;
  const int cnt = __popc(flags);
  // block exclusive scan of the per-thread counts
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = cnt;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += t;
  }
  const int in_warp = inc - cnt;
  if (lane == 31) s_warp[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    const int v = lane < kScanBlock / 32 ? s_warp[lane] : 0;
    int winc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, winc, d);
      if (lane >= d) winc += t;
    }
    if (lane < kScanBlock / 32) s_warp[lane] = winc - v;  // exclusive warp offsets
    const int aggregate = __shfl_sync(0xffffffffu, winc, 31);
    // decoupled look-back, 32 predecessors per round (status 1 = block aggregate, 2 = inclusive prefix)
    int prefix = 0;
    volatile unsigned long long *vd = desc + 1;
    if (bid == 0) {
      if (lane == 0) vd[0] = (2ull << 32) | static_cast<uint32_t>(aggregate);
    } else {
      if (lane == 0) vd[bid] = (1ull << 32) | static_cast<uint32_t>(aggregate);
      int j = static_cast<int>(bid) - 1;  // lane l inspects block j - l
      while (true) {
        const int b = j - lane;
        const unsigned long long d = b >= 0 ? vd[b] : (2ull << 32);  // before block 0: inclusive prefix 0
        const uint32_t st = static_cast<uint32_t>(d >> 32);
        const unsigned incl = __ballot_sync(0xffffffffu, st == 2);
        const unsigned ready = __ballot_sync(0xffffffffu, st != 0);
        const int last = incl ? __ffs(incl) - 1 : 31;                     // nearest inclusive prefix (or all 32)
        const unsigned need = last == 31 ? 0xffffffffu : ((2u << last) - 1u);
        if ((ready & need) != need) continue;                             // a needed predecessor has not posted yet
        int val = lane <= last ? static_cast<int>(static_cast<uint32_t>(d)) : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) val += __shfl_xor_sync(0xffffffffu, val, o);
        prefix += val;
        if (incl) break;
        j -= 32;
      }
      if (lane == 0) vd[bid] = (2ull << 32) | static_cast<uint32_t>(prefix + aggregate);
    }
    if (lane == 0) {
      s_prefix = prefix;
      if (bid == gridDim.x - 1) {
        const int total = prefix + aggregate;
        num_voxels[0] = total < max_voxels ? total : max_voxels;  // voxelize_op.cc:61-64 cap
      }
    }
  }
  __syncthreads();
  int rank = s_prefix + s_warp[wid] + in_warp;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    if (!((flags >> k) & 1u)) continue;
    const int v = rank < max_voxels ? rank : -1;
    ++rank;
    slot_vox[slot[k]] = v;
    if (v >= 0) {
      const int cell = static_cast<int>(entry[k] >> 32);
      const int cx = cell % g.gx;
      const int r = cell / g.gx;
      int32_t *c = coords + static_cast<size_t>(v) * coord_stride;
      if (coord_off) c[0] = batch_id;
      c[coord_off + 0] = r / g.gy;  // (z, y, x) order, voxelize_op.cc:66-69
      c[coord_off + 1] = r % g.gy;
      c[coord_off + 2] = cx;
    }
  }
}

// ---------------------------------------------------------------- K3
__global__ void __launch_bounds__(256) vox_slots_kernel(const int32_t *__restrict__ pt_slot,
                                                        const int32_t *__restrict__ slot_vox, int n, int P, int C,
                                                        int32_t *__restrict__ count, int32_t *__restrict__ cand,
                                                        int32_t *__restrict__ ovf) {
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int slot = pt_slot[i];
  if (slot < 0) return;
  const int v = slot_vox[slot];
  if (v < 0) return;
  // One atomic per point: arrival number inside the voxel.  The first C arrivals are simply recorded (K3b orders them);
  // on the C3 frame many points sit in voxels of 11 .. 42 points, where an all-cascade version serialises ~c x P / 2
  // dependent same-line atomics per such voxel.
  if (C > 0) {
    const int a = atomicAdd(count + v, 1);
    if (a < C) {
      cand[static_cast<size_t>(v) * C + a] = i;
      return;
    }
  }
  // Voxels with more than C points (dense clusters): the P smallest indices of the overflow arrivals, by a cascade of
  // atomicMin - slot s converges to the (s+1)-th smallest under any interleaving.  Every entry only ever decreases, so
  // once the LAST entry is below i, i can never be among the P smallest, and the leading levels already below i are
  // skipped after one round of independent loads.
  int32_t *L = ovf + static_cast<size_t>(v) * P;
  if (__ldcg(L + P - 1) < i) return;
  int s = 0;
  for (int s0 = 0; s0 < P; s0 += 8) {
    int val[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) val[k] = (s0 + k < P) ? __ldcg(L + s0 + k) : kInf;
    // lists are not guaranteed sorted mid-flight: only the LEADING run of "already smaller" levels may be skipped
    int lead = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) lead += (lead == k && val[k] < i) ? 1 : 0;
    s += lead;
    if (lead < 8) break;
  }
  if (s >= P) return;
  int cur = i;
  for (; s < P; ++s) {
    // plain (L1-cached, possibly stale) read: entries only shrink, so a stale "already smaller" is still true and the
    // atomic can be skipped at L1 latency; a stale "larger" merely costs the atomic, which returns the fresh value
    // (with ld.cg here every level walked would cost an L2 round trip)
    if (L[s] < cur) continue;
    const int old = atomicMin(&L[s], cur);
    if (old == kInf) break;     // landed in a free slot
    if (old > cur) cur = old;   // displaced a larger index: carry it down
  }
}

// ---------------------------------------------------------------- K3b
// lists[v][0..P) = the P smallest point indices of voxel v in ascending order (INF padding) - the CPU kernel's "first P
// points in input order" (voxelize_op.cc:71-79) - selected from the recorded arrivals (plus, for voxels beyond C points,
// the cascade's P survivors: the P smallest overall are among the first C arrivals or the P smallest of the rest).
// One thread per (voxel, slot): it ranks its share of the candidates (indices are distinct, so ranks are unique) and
// stores each candidate of rank < P at lists[v][rank]; slots no candidate reaches get INF.
__global__ void __launch_bounds__(256) vox_select_kernel(const int32_t *__restrict__ count, const int32_t *__restrict__ cand,
                                                         const int32_t *__restrict__ ovf, int V, int P, int C,
                                                         int32_t *__restrict__ lists) {
  pdl_trigger();
  pdl_wait();
  const long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (q >= static_cast<long long>(V) * P) return;
  const int v = static_cast<int>(q / P), s = static_cast<int>(q - static_cast<long long>(v) * P);
  const int cnt = __ldg(count + v);
  const int m = cnt < C ? cnt : C;
  const int total = m + (cnt > C ? P : 0);
  const int32_t *cv = cand + static_cast<size_t>(v) * C, *ov = ovf + static_cast<size_t>(v) * P;
  if (s >= (cnt < P ? cnt : P)) lists[q] = kInf;  // cnt > C >= P: every slot is reached
  // (both arrays were completed by the previous launch: read-only loads, four comparisons in flight)
  for (int j = s; j < total; j += P) {
    const int x = j < m ? __ldg(cv + j) : __ldg(ov + (j - m));
    if (x == kInf) continue;
    int rank = 0;
    int k = 0;
    for (; k + 4 <= m; k += 4) {
      const int4 c4 = __ldg(reinterpret_cast<const int4 *>(cv + k));  // C is a multiple of 4, rows are 16-byte aligned
      rank += (c4.x < x) + (c4.y < x) + (c4.z < x) + (c4.w < x);
    }
    for (; k < m; ++k) rank += (__ldg(cv + k) < x) ? 1 : 0;
    for (k = m; k < total; ++k) rank += (__ldg(ov + (k - m)) < x) ? 1 : 0;
    if (rank < P) lists[static_cast<size_t>(v) * P + rank] = x;
  }
}

// ---------------------------------------------------------------- K4
__device__ __forceinline__ void st_stream(float4 *p, float4 v) { __stcs(p, v); }

constexpr int kWriteRows = 256;  // (voxel, slot) rows per block of the writer

// One block = 256 consecutive (voxel, slot) rows of voxels[V, P, F]: each thread reads ITS row's point index (coalesced)
// and copies the F floats of that point (or zeros) into shared memory; then the block streams the 256 * F floats out as
// float4, fully coalesced - every byte of the output is written exactly once, no integer division on the store path.
__global__ void __launch_bounds__(kWriteRows) vox_write_kernel(const float *__restrict__ points, int F, int P, int V,
                                                               const int32_t *__restrict__ lists,
                                                               const int32_t *__restrict__ num_voxels_dev,
                                                               float *__restrict__ voxels, int32_t *__restrict__ coords,
                                                               int32_t *__restrict__ npv, long long rows_total) {
  extern __shared__ __align__(16) float s_stage[];  // [kWriteRows][F]
  pdl_trigger();
  pdl_wait();
  const int tid = threadIdx.x;
  const long long r0 = static_cast<long long>(blockIdx.x) * kWriteRows;
  const int nrows = static_cast<int>(min(static_cast<long long>(kWriteRows), rows_total - r0));
  if (tid < nrows) {
    const int idx = __ldg(lists + r0 + tid);
    float *dst = s_stage + tid * F;
    if (idx != kInf) {
      const float *src = points + static_cast<size_t>(idx) * F;
      for (int f = 0; f < F; ++f) dst[f] = __ldg(src + f);
    } else {
      for (int f = 0; f < F; ++f) dst[f] = 0.f;
    }
  }
  __syncthreads();
  const int cnt = nrows > 0 ? nrows * F : 0;
  float *out = voxels + r0 * F;  // r0 is a multiple of 256: 16-byte aligned whenever `voxels` is
  const int c4 = cnt >> 2;
  for (int q = tid; q < c4; q += kWriteRows) st_stream(reinterpret_cast<float4 *>(out) + q, reinterpret_cast<const float4 *>(s_stage)[q]);
  for (int e = (c4 << 2) + tid; e < cnt; e += kWriteRows) out[e] = s_stage[e];
  // per-voxel outputs: one thread per voxel, strided over the grid
  const long long gtid = static_cast<long long>(blockIdx.x) * kWriteRows + tid;
  for (long long v = gtid; v < V; v += static_cast<long long>(gridDim.x) * kWriteRows) {
    int c = 0;
    for (int s = 0; s < P; ++s) c += (__ldg(lists + static_cast<size_t>(v) * P + s) != kInf);
    npv[v] = c;
    if (v >= num_voxels_dev[0]) {
      coords[v * 3 + 0] = 0;
      coords[v * 3 + 1] = 0;
      coords[v * 3 + 2] = 0;
    }
  }
}

// Fused VoxelMean writer (voxel_encoder.py:49-57): mean over the kept points, summed in slot order.
__global__ void __launch_bounds__(256) vox_mean_kernel(const float *__restrict__ points, int F, int P, int V,
                                                       const int32_t *__restrict__ lists,
                                                       const int32_t *__restrict__ num_voxels_dev,
                                                       float *__restrict__ mean, int32_t *__restrict__ coors4,
                                                       int32_t *__restrict__ npv) {
  pdl_trigger();
  pdl_wait();
  const long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (q >= static_cast<long long>(V) * F) return;
  const int v = static_cast<int>(q / F), f = static_cast<int>(q - static_cast<long long>(v) * F);
  float s = 0.f;
  int cnt = 0;
  for (int k = 0; k < P; ++k) {
    const int idx = lists[static_cast<size_t>(v) * P + k];
    if (idx == kInf) break;  // lists are ascending with INF padding
    s += __ldg(points + static_cast<size_t>(idx) * F + f);
    ++cnt;
  }
  const bool live = v < num_voxels_dev[0];
  mean[q] = live ? __fdiv_rn(s, static_cast<float>(cnt)) : 0.f;
  if (f == 0) {
    npv[v] = cnt;
    if (!live) {
      int4 z = make_int4(0, 0, 0, 0);
      *reinterpret_cast<int4 *>(coors4 + static_cast<size_t>(v) * 4) = z;
    }
  }
}

__global__ void __launch_bounds__(256) voxel_mean_kernel(const float *__restrict__ voxels,
                                                         const int32_t *__restrict__ npv,
                                                         const int32_t *__restrict__ nv_dev, int cap, int P, int F,
                                                         float *__restrict__ mean) {
  const long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (q >= static_cast<long long>(cap) * F) return;
  const int v = static_cast<int>(q / F), f = static_cast<int>(q - static_cast<long long>(v) * F);
  if (nv_dev && v >= nv_dev[0]) {
    mean[q] = 0.f;
    return;
  }
  float s = 0.f;
  for (int k = 0; k < P; ++k) s += voxels[(static_cast<size_t>(v) * P + k) * F + f];
  mean[q] = __fdiv_rn(s, static_cast<float>(npv[v]));
}

int check_geom(const float *vs, const float *pcr, int64_t n, int F, int P, int V, VoxGeom *g) {
  if (!vs || !pcr || n < 0 || F < 3 || P < 1 || V < 1) return P3D_ERR_INVALID_ARG;
  if (n > kMaxRows) return P3D_ERR_UNSUPPORTED;  // the cell hash holds 2 n entries (next_pow2 saturates beyond 2^31)
  g->min_x = pcr[0];
  g->min_y = pcr[1];
  g->min_z = pcr[2];
  g->vs_x = vs[0];
  g->vs_y = vs[1];
  g->vs_z = vs[2];
  // grid = round((max - min) / size) in fp32, voxelize_op.cc:97-102
  g->gx = static_cast<int>(roundf((pcr[3] - pcr[0]) / vs[0]));
  g->gy = static_cast<int>(roundf((pcr[4] - pcr[1]) / vs[1]));
  g->gz = static_cast<int>(roundf((pcr[5] - pcr[2]) / vs[2]));
  if (g->gx < 1 || g->gy < 1 || g->gz < 1) return P3D_ERR_INVALID_ARG;
  if (static_cast<double>(g->gx) * g->gy * g->gz >= 2147483648.0) return P3D_ERR_UNSUPPORTED;
  if (static_cast<long long>(V) * P * F >= (1ll << 40)) return P3D_ERR_UNSUPPORTED;
  return P3D_OK;
}

int run_front(const float *points, int n, int F, const VoxGeom &g, int P, int V, const VoxWs &w, int32_t *coords,
              int coord_stride, int coord_off, int batch_id, int32_t *num_voxels, cudaStream_t st) {
  const size_t n_t16 = static_cast<size_t>(w.cap) / 2;
  const size_t n_d16 = (static_cast<size_t>(w.nblocks) + 1 + 1) / 2;  // carve() pads to 256 B
  const size_t n_l16 = (static_cast<size_t>(V) * P + 3) / 4;
  P3D_CUDA_CHECK(launch_pdl(vox_init_kernel, dim3(num_sms() * 4), dim3(256), 0, st, reinterpret_cast<uint4 *>(w.table), n_t16,
                            reinterpret_cast<uint4 *>(w.desc), n_d16, reinterpret_cast<uint4 *>(w.ovf), n_l16,
                            reinterpret_cast<uint4 *>(w.count), (static_cast<size_t>(V) + 3) / 4));
  if (n > 0) {
    P3D_CUDA_CHECK(launch_pdl(vox_insert_kernel, dim3(div_up(n, 256)), dim3(256), 0, st, points, n, F, g, w.table,
                              w.cap - 1, w.shift, w.pt_slot));
    P3D_CUDA_CHECK(launch_pdl(vox_rank_kernel, dim3(w.nblocks), dim3(kScanBlock), 0, st, w.table, w.pt_slot, n, V, g, w.desc,
                              w.slot_vox, coords, coord_stride, coord_off, batch_id, num_voxels));
    P3D_CUDA_CHECK(launch_pdl(vox_slots_kernel, dim3(div_up(n, 256)), dim3(256), 0, st, w.pt_slot, w.slot_vox, n, P, w.C,
                              w.count, w.cand, w.ovf));
  } else {
    P3D_CUDA_CHECK(cudaMemsetAsync(num_voxels, 0, sizeof(int32_t), st));
  }
  if (w.C > 0)
    P3D_CUDA_CHECK(launch_pdl(vox_select_kernel, dim3(div_up(static_cast<long long>(V) * P, 256)), dim3(256), 0, st, w.count, w.cand,
                              w.ovf, V, P, w.C, w.lists));
  return P3D_OK;
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" size_t p3d_hard_voxelize_workspace_bytes(int64_t num_points, int max_points, int max_voxels) {
  if (num_points < 0 || num_points > kMaxRows || max_points < 1 || max_voxels < 1) return 0;
  return carve(nullptr, num_points, max_points, max_voxels).bytes;
}

extern "C" int p3d_hard_voxelize(const float *points, int64_t num_points, int num_point_dim,
                                 const float *voxel_size_host, const float *point_cloud_range_host, int max_points,
                                 int max_voxels, float *voxels, int32_t *coords, int32_t *num_points_per_voxel,
                                 int32_t *num_voxels, void *workspace, size_t workspace_bytes,
                                 p3d_stream_t stream) {
  VoxGeom g;
  int rc = check_geom(voxel_size_host, point_cloud_range_host, num_points, num_point_dim, max_points, max_voxels, &g);
  if (rc) return rc;
  if ((!points && num_points) || !voxels || !coords || !num_points_per_voxel || !num_voxels || !workspace)
    return P3D_ERR_INVALID_ARG;
  if ((reinterpret_cast<uintptr_t>(voxels) & 15) || (reinterpret_cast<uintptr_t>(workspace) & 255))
    return P3D_ERR_INVALID_ARG;
  const VoxWs w = carve(workspace, num_points, max_points, max_voxels);
  if (workspace_bytes < w.bytes) return P3D_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int n = static_cast<int>(num_points);
  rc = run_front(points, n, num_point_dim, g, max_points, max_voxels, w, coords, 3, 0, 0, num_voxels, st);
  if (rc) return rc;
  const long long rows_total = static_cast<long long>(max_voxels) * max_points;
  const long long blocks = (rows_total + kWriteRows - 1) / kWriteRows;
  const size_t stage = static_cast<size_t>(kWriteRows) * num_point_dim * sizeof(float);
  if (stage > 48 * 1024) return P3D_ERR_UNSUPPORTED;  // F <= 48 point features
  P3D_CUDA_CHECK(launch_pdl(vox_write_kernel, dim3(static_cast<unsigned int>(blocks)), dim3(kWriteRows), stage, st, points,
                            num_point_dim, max_points, max_voxels, w.lists, num_voxels, voxels, coords,
                            num_points_per_voxel, rows_total));
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}

extern "C" int p3d_voxelize_mean(const float *points, int64_t num_points, int num_point_dim,
                                 const float *voxel_size_host, const float *point_cloud_range_host, int max_points,
                                 int max_voxels, int batch_id, float *mean, int32_t *coors4,
                                 int32_t *num_points_per_voxel, int32_t *num_voxels, void *workspace,
                                 size_t workspace_bytes, p3d_stream_t stream) {
  VoxGeom g;
  int rc = check_geom(voxel_size_host, point_cloud_range_host, num_points, num_point_dim, max_points, max_voxels, &g);
  if (rc) return rc;
  if ((!points && num_points) || !mean || !coors4 || !num_points_per_voxel || !num_voxels || !workspace)
    return P3D_ERR_INVALID_ARG;
  if ((reinterpret_cast<uintptr_t>(coors4) & 15) || (reinterpret_cast<uintptr_t>(workspace) & 255))
    return P3D_ERR_INVALID_ARG;
  const VoxWs w = carve(workspace, num_points, max_points, max_voxels);
  if (workspace_bytes < w.bytes) return P3D_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  rc = run_front(points, static_cast<int>(num_points), num_point_dim, g, max_points, max_voxels, w, coors4, 4, 1,
                 batch_id, num_voxels, st);
  if (rc) return rc;
  const long long threads = static_cast<long long>(max_voxels) * num_point_dim;
  P3D_CUDA_CHECK(launch_pdl(vox_mean_kernel, dim3(div_up(threads, 256)), dim3(256), 0, st, points, num_point_dim, max_points,
                            max_voxels, w.lists, num_voxels, mean, coors4, num_points_per_voxel));
  return P3D_OK;
}

extern "C" int p3d_voxel_mean(const float *voxels, const int32_t *num_points_per_voxel,
                              const int32_t *num_voxels_dev, int num_voxels_cap, int max_points, int num_point_dim,
                              float *mean, p3d_stream_t stream) {
  if (!voxels || !num_points_per_voxel || !mean || num_voxels_cap < 0 || max_points < 1 || num_point_dim < 1)
    return P3D_ERR_INVALID_ARG;
  if (num_voxels_cap == 0) return P3D_OK;
  const long long threads = static_cast<long long>(num_voxels_cap) * num_point_dim;
  voxel_mean_kernel<<<div_up(threads, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      voxels, num_points_per_voxel, num_voxels_dev, num_voxels_cap, max_points, num_point_dim, mean);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
