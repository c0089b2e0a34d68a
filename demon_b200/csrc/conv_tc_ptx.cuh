// PTX wrappers of the tensor-core convolution kernel (sm_90a): mbarrier, TMA / bulk copies, wgmma.
#pragma once
#include <cuda.h>
#include <cstdint>

namespace demon {
namespace {

constexpr long long kTimeoutCycles = 4000000000ll;   // ~2 s at 1.9 GHz

// ---- PTX wrappers ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.shared::cta.b64 st, [%0];\n}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n}" ::"r"(bar), "r"(bytes) : "memory");
}
// Bounded wait: a pipeline bug must not hang the GPU; on timeout the error flag is raised and the kernel runs to
// completion with garbage (the host checks the flag in tests).
__device__ __forceinline__ bool mbar_try(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n.reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n}"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done != 0;
}
// non-blocking probe (try_wait may suspend the thread for a hardware time-out when the phase is still pending)
__device__ __forceinline__ bool mbar_test(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n.reg .pred p;\n"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n}"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done != 0;
}
__device__ __noinline__ bool mbar_wait_slow(uint32_t bar, uint32_t parity, int* err) {
  const long long t0 = clock64();
  for (;;) {
    for (int i = 0; i < 64; ++i)
      if (mbar_try(bar, parity)) return true;
    if (*reinterpret_cast<volatile int*>(err) != 0) return false;   // somebody already timed out: drain quickly
    if (clock64() - t0 > kTimeoutCycles) {
      atomicExch(err, 1);
      return false;
    }
  }
}
__device__ __forceinline__ bool mbar_wait(uint32_t bar, uint32_t parity, int* err) {
  if (mbar_try(bar, parity)) return true;
  return mbar_wait_slow(bar, parity, err);
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous wgmma region
__device__ __forceinline__ void reg_fence(float& x) { asm volatile("" : "+f"(x)::"memory"); }

// Shared-memory matrix descriptor (sm_90 wgmma), K-major operand with 128-byte swizzle: rows of 128 bytes, 8-row groups
// 1024 bytes apart (stride byte offset), layout type 1 = SWIZZLE_128B.  Advancing the start address by 32 bytes selects
// the next K = 8 slice inside the swizzled rows.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);   // start address, bits [0,14)
  d |= (uint64_t)1 << 16;                        // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;              // stride byte offset, bits [32,46)
  d |= (uint64_t)1 << 62;                        // SWIZZLE_128B
  return d;
}

// elect.sync: exactly one lane of the (converged) warp gets `true`.  Unlike `lane == 0`, the compiler then KNOWS the
// region runs with a single active thread and emits the uniform-datapath instructions (UTMALDG, UBLKCP, ...)
// directly instead of wrapping each one in a per-thread serialisation loop.
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred;
  asm volatile("{\n.reg .b32 rx;\n.reg .pred px;\nelect.sync rx|px, 0xffffffff;\nselp.b32 %0, 1, 0, px;\n}" : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
}  // namespace
}  // namespace demon
