// Shared helpers for libp3d_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "p3d_b200.h"

namespace p3d {

extern thread_local int g_last_cuda_error;

inline int cuda_fail(cudaError_t e) {
  g_last_cuda_error = static_cast<int>(e);
  return P3D_ERR_CUDA;
}

#define P3D_CUDA_CHECK(expr)                                \
  do {                                                      \
    cudaError_t _e = (expr);                                \
    if (_e != cudaSuccess) return ::p3d::cuda_fail(_e);     \
  } while (0)
#define P3D_LAUNCH_CHECK() P3D_CUDA_CHECK(cudaGetLastError())

constexpr size_t kAlign = 256;
inline size_t align_up(size_t x, size_t a = kAlign) { return (x + a - 1) / a * a; }

// Sequential carve-out of a caller-provided workspace (also used to size it).
struct Carver {
  char *base;
  size_t off = 0;
  explicit Carver(void *p) : base(static_cast<char *>(p)) {}
  template <typename T>
  T *take(size_t count) {
    T *r = reinterpret_cast<T *>(base + off);
    off += align_up(count * sizeof(T));
    return r;
  }
};

inline unsigned int div_up(long long a, long long b) { return static_cast<unsigned int>((a + b - 1) / b); }
// Smallest power of two >= x, saturating at 2^31 (computed in 64 bits: a 32-bit accumulator wraps to 0 for x > 2^31 and
// the loop never ends - ADVICE r1).  Callers reject row counts above kMaxRows before sizing a table with it.
constexpr int64_t kMaxRows = 1ll << 29;  // hash tables hold 2x the rows: 2^30 64-bit entries at most
inline uint32_t next_pow2(uint64_t x) {
  uint64_t p = 1;
  while (p < x && p < (1ull << 31)) p <<= 1;
  return static_cast<uint32_t>(p);
}

// Multiprocessors of the current device (persistent grids are sized by it; 132 on an H100 SXM).
inline int num_sms() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1)
    return 132;
  return n;
}

// Programmatic dependent launch: the grid may be scheduled while its predecessor in the stream drains.  Every kernel
// launched this way executes pdl_wait() before it touches global memory (and pdl_trigger() first, so that ITS successor
// can be scheduled early as well).  P3D_PDL=0 falls back to plain stream order.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
bool pdl_enabled();
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// Decoupled look-back across the tiles of a single-pass scan, 32 predecessors per round.  Called by all 32 lanes of one
// warp of tile `bid` (tiles numbered in scan order, e.g. by an atomic ticket) with that tile's aggregate; returns the sum
// of the aggregates of tiles [0, bid) in every lane and publishes the tile's inclusive prefix.  desc[b] =
// (status << 32 | value): status 0 = not posted yet, 1 = tile aggregate, 2 = inclusive prefix; zero before the launch.
__device__ __forceinline__ int lookback_exclusive_prefix(unsigned long long *desc, unsigned int bid, int aggregate) {
  const int lane = threadIdx.x & 31;
  int prefix = 0;
  volatile unsigned long long *vd = desc;
  if (bid == 0) {
    if (lane == 0) vd[0] = (2ull << 32) | static_cast<uint32_t>(aggregate);
    return 0;
  }
  if (lane == 0) vd[bid] = (1ull << 32) | static_cast<uint32_t>(aggregate);
  int j = static_cast<int>(bid) - 1;  // lane l inspects tile j - l
  while (true) {
    const int b = j - lane;
    const unsigned long long d = b >= 0 ? vd[b] : (2ull << 32);  // before tile 0: inclusive prefix 0
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
  return prefix;
}

__device__ __forceinline__ uint32_t hash32(uint32_t k) {
  k *= 0x9E3779B1u;  // Fibonacci hashing; callers take the top bits
  return k;
}

}  // namespace p3d
