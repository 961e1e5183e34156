// Shared helpers for the mt3_b200 CUDA library (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <string>

#include "../../include/mt3_b200.h"

namespace mt3 {

// thread-local last-error text behind mt3_last_error()
std::string& last_error();
int fail(int code, const char* fmt, ...);

extern std::atomic<uint64_t> g_launch_count;
inline void count_launch(uint64_t n = 1) { g_launch_count.fetch_add(n, std::memory_order_relaxed); }

#define MT3_CUDA_CHECK(expr)                                                                   \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess)                                                                     \
      return ::mt3::fail(MT3_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr,            \
                         cudaGetErrorString(_e));                                              \
  } while (0)

#define MT3_LAUNCH_CHECK()                                                                     \
  do {                                                                                         \
    cudaError_t _e = cudaGetLastError();                                                       \
    if (_e != cudaSuccess)                                                                     \
      return ::mt3::fail(MT3_ERR_CUDA, "%s:%d kernel launch -> %s", __FILE__, __LINE__,        \
                         cudaGetErrorString(_e));                                              \
    ::mt3::count_launch();                                                                     \
  } while (0)

#define MT3_REQUIRE(cond, code, ...)                                                           \
  do {                                                                                         \
    if (!(cond)) return ::mt3::fail(code, __VA_ARGS__);                                        \
  } while (0)

#define MT3_TRY(expr)            \
  do {                           \
    int _r = (expr);             \
    if (_r != MT3_OK) return _r; \
  } while (0)

// Raises Kernel's dynamic shared-memory limit to `bytes` before its first launch: once per kernel instantiation, as each
// instantiation of this template has its own flag.
template <auto Kernel>
inline int set_max_dynamic_smem(int bytes) {
  static bool done = false;
  if (!done) {
    MT3_CUDA_CHECK(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    done = true;
  }
  return MT3_OK;
}

inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }
inline int cdiv(int a, int b) { return (a + b - 1) / b; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Programmatic dependent launch (PDL).  pdl_wait(): block until every prerequisite grid has completed and
// its memory is visible; nothing a predecessor produces may be read, and nothing it may still read may be
// written, before this.  pdl_trigger(): let the dependent grid start launching (it still waits at its own
// pdl_wait()).  Both are no-ops for kernels launched without the PDL attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Launch with (or without) the programmatic-stream-serialization attribute.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl,
                                 Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// Launch with a thread-block cluster of (1, cluster_y, 1) CTAs, with (or without) the programmatic-stream-serialization
// attribute.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                         unsigned cluster_y, bool pdl, Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1;
  attr[0].val.clusterDim.y = cluster_y;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 2 : 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// d.x = a * b.x + d.x, d.y = a * b.y + d.y: two IEEE fp32 FMAs.
__device__ __forceinline__ void ffma2(float2& d, float a, float2 b) {
  d.x = fmaf(a, b.x, d.x);
  d.y = fmaf(a, b.y, d.y);
}

// x = hi + lo with hi = x truncated to tf32 (what a tf32 wgmma reads), lo = x - hi (exact in fp32).
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  hi = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
  lo = x - hi;
}

}  // namespace mt3
