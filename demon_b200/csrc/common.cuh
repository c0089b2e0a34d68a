// Shared helpers of the demon_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <string>

#include "../../include/demon_b200.h"

namespace demon {

// ---- error plumbing: C ABI returns a code, message kept thread-local -------------------------
std::string& last_error_ref();
int fail(int code, const char* fmt, ...);
extern std::atomic<int64_t> g_launch_count;

#define DEMON_CHECK_CUDA(expr)                                                              \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess)                                                                  \
      return ::demon::fail(DEMON_E_CUDA, "%s:%d: %s failed: %s", __FILE__, __LINE__, #expr, \
                           cudaGetErrorString(_e));                                         \
  } while (0)

// Every kernel launch goes through this: counts launches (gpu_launches in bench.py) and turns a
// launch failure into an error code, like _CHECK_CUDA_ERROR did in the reference
// (lmbspecialops/src/cuda_helper.h:25-35) but without throwing across the C ABI.
#define DEMON_LAUNCH_CHECK()                                                                    \
  do {                                                                                          \
    ::demon::g_launch_count.fetch_add(1, std::memory_order_relaxed);                            \
    cudaError_t _e = cudaPeekAtLastError();                                                     \
    if (_e != cudaSuccess) {                                                                    \
      cudaGetLastError();                                                                       \
      return ::demon::fail(DEMON_E_CUDA, "%s:%d: kernel launch failed: %s", __FILE__, __LINE__, \
                           cudaGetErrorString(_e));                                             \
    }                                                                                           \
  } while (0)

#define DEMON_REQUIRE(cond, ...)                                   \
  do {                                                             \
    if (!(cond)) return ::demon::fail(DEMON_E_INVALID, __VA_ARGS__); \
  } while (0)

// ---- programmatic dependent launch (PDL) ------------------------------------------------------
// The pipeline is a chain of ~270 short kernels on one stream.  A kernel launched through launch_pdl() may become
// resident while its predecessor is still draining: its prologue (barrier init, tensor-map prefetch,
// parameter loads, the first weight blocks) overlaps the predecessor's tail, and the launch latency disappears from the
// chain.  Contract: such a kernel calls pdl_wait() before it reads anything an earlier kernel wrote and before its first
// global store (buffers are reused along the chain), and every kernel calls pdl_launch_dependents() early so that its
// successor may start.  DEMON_PDL=0 falls back to plain stream order (for A/B measurements).
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---- IEEE ops without FMA contraction ---------------------------------------------------------
// The geometry ops restate x86 code compiled without FMA; using the _rn intrinsics keeps nvcc from
// contracting a*b+c so the float results match the CPU oracle operation for operation.
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double fmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double fadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double fsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double fdiv(double a, double b) { return __ddiv_rn(a, b); }

}  // namespace demon
