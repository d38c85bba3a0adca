// wgmma.mma_async wrappers (sm_90a): D (fp32 registers, m64nN fragment) += A (shared-memory descriptor) x B (descriptor).
// One specialisation per N used by the kernels; scale_d = 0 overwrites D instead of accumulating.
// Fragment of thread t of the warpgroup (warp w = t / 32, lane l): d[4j + 2h + e] = D[16w + l/4 + 8h][8j + 2(l%4) + e].
#pragma once
#include <stdint.h>

#define P3D_ACC4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define P3D_ACC8(i) P3D_ACC4(i), P3D_ACC4(i + 4)
#define P3D_ACC16(i) P3D_ACC8(i), P3D_ACC8(i + 8)

namespace p3d {
namespace wg {

template <int N>
__device__ __forceinline__ void mma_f16(float *d, uint64_t a, uint64_t b, uint32_t scale_d);
template <int N>
__device__ __forceinline__ void mma_tf32(float *d, uint64_t a, uint64_t b, uint32_t scale_d);

template <>
__device__ __forceinline__ void mma_f16<16>(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\twgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
               : P3D_ACC8(0)
               : "l"(a), "l"(b), "r"(scale_d));
}

template <>
__device__ __forceinline__ void mma_f16<32>(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\twgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
               : P3D_ACC16(0)
               : "l"(a), "l"(b), "r"(scale_d));
}

template <>
__device__ __forceinline__ void mma_f16<64>(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
               : P3D_ACC16(0), P3D_ACC16(16)
               : "l"(a), "l"(b), "r"(scale_d));
}

template <>
__device__ __forceinline__ void mma_f16<128>(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
               : P3D_ACC16(0), P3D_ACC16(16), P3D_ACC16(32), P3D_ACC16(48)
               : "l"(a), "l"(b), "r"(scale_d));
}

template <>
__device__ __forceinline__ void mma_tf32<16>(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\twgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}"
               : P3D_ACC8(0)
               : "l"(a), "l"(b), "r"(scale_d));
}

template <>
__device__ __forceinline__ void mma_tf32<32>(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\twgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
               : P3D_ACC16(0)
               : "l"(a), "l"(b), "r"(scale_d));
}

template <>
__device__ __forceinline__ void mma_tf32<64>(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
               : P3D_ACC16(0), P3D_ACC16(16)
               : "l"(a), "l"(b), "r"(scale_d));
}

template <>
__device__ __forceinline__ void mma_tf32<128>(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
               : P3D_ACC16(0), P3D_ACC16(16), P3D_ACC16(32), P3D_ACC16(48)
               : "l"(a), "l"(b), "r"(scale_d));
}

}  // namespace wg
}  // namespace p3d

#undef P3D_ACC16
#undef P3D_ACC8
#undef P3D_ACC4
