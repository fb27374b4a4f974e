// Raw PTX wrappers for the Hopper asynchronous machinery (mbarrier, bulk copy, wgmma, elect.sync), shared by the wgmma
// kernels (tc5_kernels.cu: Spiral first dimension; dpir_gemm.cu: DoublePIR offline GEMMs).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "tc5_layout.cuh"

namespace b200pir {
namespace tc5 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// Bounded wait: a protocol error must surface as a launch failure (trap), never as a hung GPU.  Plain try_wait in a spin loop
// (no suspend-time hint: a hinted wait may park the thread for long quanta, and every stage hand-off of the pipeline goes
// through one of these); the bound is on elapsed clocks (~20 s), checked every 1024 polls.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  long long t0 = 0;
  for (uint32_t tries = 0;; tries++) {
    uint32_t done;
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P1;\n\t"
        "}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) return;
    if ((tries & 1023u) == 1023u) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 40000000000ll) asm volatile("trap;");
    }
  }
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// one lane of the (converged) warp
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// The wait names no registers, so without this the compiler may move reads of the accumulators above it: every accumulator
// register goes through an (empty) asm that is ordered after the wait.
template <int N>
__device__ __forceinline__ void wgmma_fence_operands(uint32_t (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; i++) asm volatile("" : "+r"(d[i])::"memory");
}

#define TC5_R8(v, o) "+r"(v[o]), "+r"(v[o + 1]), "+r"(v[o + 2]), "+r"(v[o + 3]), "+r"(v[o + 4]), "+r"(v[o + 5]), "+r"(v[o + 6]), "+r"(v[o + 7])
// D (64 x 128, s32 fragment of the warpgroup) += A (64 x 32 u8, K-major) * B (128 x 32 u8, K-major)^T, no saturation
__device__ __forceinline__ void wgmma_m64n128k32_u8(uint32_t (&d)[64], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.u8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1;"
      : TC5_R8(d, 0), TC5_R8(d, 8), TC5_R8(d, 16), TC5_R8(d, 24), TC5_R8(d, 32), TC5_R8(d, 40), TC5_R8(d, 48), TC5_R8(d, 56)
      : "l"(desc_a), "l"(desc_b)
      : "memory");
}
// D (64 x 32) += A (64 x 32, u8 or s8) * B (32 x 32 u8)^T, wrapping modulo 2^32
template <bool A_SIGNED>
__device__ __forceinline__ void wgmma_m64n32k32(uint32_t (&d)[16], uint64_t desc_a, uint64_t desc_b) {
  if (A_SIGNED)
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.u8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, 1;"
        : TC5_R8(d, 0), TC5_R8(d, 8)
        : "l"(desc_a), "l"(desc_b)
        : "memory");
  else
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n32k32.s32.u8.u8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, 1;"
        : TC5_R8(d, 0), TC5_R8(d, 8)
        : "l"(desc_a), "l"(desc_b)
        : "memory");
}
#undef TC5_R8

__device__ __forceinline__ uint64_t shfl_xor_u64(uint64_t v, int m) {
  uint32_t lo = __shfl_xor_sync(0xffffffffu, (uint32_t)v, m), hi = __shfl_xor_sync(0xffffffffu, (uint32_t)(v >> 32), m);
  return ((uint64_t)hi << 32) | lo;
}


}  // namespace tc5
}  // namespace b200pir
