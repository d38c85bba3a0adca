// PTX helpers shared by the tensor-core kernels (sm_90a): mbarrier, cp.async(.bulk), wgmma descriptors / fences,
// the m64nN accumulator fragment, tf32 hi/lo split.
#pragma once
#include <stdlib.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace p3d {
namespace tc {

constexpr int kM = 128;       // rows of a tile: two warpgroups, 64 rows (one wgmma M) each
constexpr int kThreads = 256;  // the two warpgroups; every thread gathers, issues wgmma and runs the epilogue

__host__ __device__ constexpr int kc_of(int cin) { return cin < 16 ? cin : 16; }  // channels per pipeline stage

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
#ifndef P3D_MBAR_HINT_NS
#define P3D_MBAR_HINT_NS 20000  // suspend-time hint of mbarrier.try_wait (ns); build with -DP3D_MBAR_HINT_NS=.. to experiment
#endif
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  // try_wait with a suspend-time hint: the thread sleeps in hardware until the phase completes (or ~20 us pass)
  // instead of polling, so waiting warps do not take issue slots from the ones doing the work.
  uint32_t done;
  int spins = 0;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(static_cast<uint32_t>(P3D_MBAR_HINT_NS))
        : "memory");
    if (!done && ++spins > 200000) __trap();  // seconds: a protocol bug must not hang the GPU
  } while (!done);
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, bool valid) {
  const uint32_t sz = valid ? 16u : 0u;  // src-size 0 => 16 bytes of zeros
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// wgmma: fence before the first wgmma that touches freshly written accumulator registers, commit the issued wgmmas as
// one group, wait until at most N groups of this warp are in flight.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma
template <int R>
__device__ __forceinline__ void wg_fence_acc(float *d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// wgmma shared-memory matrix descriptor: start address, leading / stride byte offsets, layout (0 no swizzle,
// 1 SWIZZLE_128B, 2 SWIZZLE_64B, 3 SWIZZLE_32B).  K-major, no swizzle: core matrix = 8 rows x 16 B contiguous; LBO =
// distance between the two 16-byte K-chunks of one k-step, SBO = distance between 8-row groups.  K-major swizzled: LBO
// unused (1), SBO = 8 rows x row pitch; the swizzle is applied to the absolute shared-memory address, so a start
// address advanced by k-steps (or by whole rows) reads what TMA / the XOR-ing producers wrote.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t addr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout,
                                              uint32_t base_offset = 0) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((addr & 0x3ffffu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3fffu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3fffu) << 32;
  d |= static_cast<uint64_t>(base_offset & 7u) << 49;
  d |= static_cast<uint64_t>(layout) << 62;
  return d;
}
__device__ __forceinline__ uint64_t smem_desc(uint32_t addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return gmma_desc(addr, lbo_bytes, sbo_bytes, 0);
}
__device__ __forceinline__ uint64_t desc_sw128(uint32_t addr, uint32_t sbo_bytes = 1024) { return gmma_desc(addr, 16, sbo_bytes, 1); }
__device__ __forceinline__ uint64_t desc_sw64(uint32_t addr) { return gmma_desc(addr, 16, 512, 2); }

// Position of accumulator element i of an m64nN fragment inside the warpgroup's 64 x N block (wgmma.cuh).
__device__ __forceinline__ int frag_row(int i, int wg_tid) { return ((wg_tid >> 5) << 4) + ((wg_tid & 31) >> 2) + (((i >> 1) & 1) << 3); }
__device__ __forceinline__ int frag_col(int i, int wg_tid) { return ((i >> 2) << 3) + ((wg_tid & 3) << 1) + (i & 1); }

__device__ __forceinline__ void split_tf32(float x, float &hi, float &lo) {
  uint32_t h;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(x));
  hi = __uint_as_float(h);
  const float r = x - hi;  // exact in fp32
  uint32_t l;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(r));
  lo = __uint_as_float(l);
}


// split-K factor of the tensor-core sparse conv (taps spread over this many CTAs per 128-row tile)
inline int splits_for(int Cout) {
  // tuning hooks (not a public knob): P3D_SPLITS_128 / P3D_SPLITS_64 / P3D_SPLITS_32 override the defaults
  static const int s128 = getenv("P3D_SPLITS_128") ? atoi(getenv("P3D_SPLITS_128")) : 2;
  static const int s64 = getenv("P3D_SPLITS_64") ? atoi(getenv("P3D_SPLITS_64")) : 2;
  static const int s32 = getenv("P3D_SPLITS_32") ? atoi(getenv("P3D_SPLITS_32")) : 1;
  const int v = Cout >= 128 ? s128 : (Cout >= 64 ? s64 : s32);
  return v < 1 ? 1 : (v > 8 ? 8 : v);
}

}  // namespace tc
}  // namespace p3d
