// aph_common.cuh -- shared helpers for libaphb200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>

#include "../../include/aphb200.h"

namespace aph {

void set_error(const char* fmt, ...);          // defined in api.cu (thread-local message)
extern std::atomic<long long> g_launches;      // kernels launched by this library

inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define APH_CUDA_OK(expr)                                                                       \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess) {                                                                    \
      aph::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));      \
      return 1;                                                                                 \
    }                                                                                           \
  } while (0)

#define APH_REQUIRE(cond, ...)                                                                  \
  do {                                                                                          \
    if (!(cond)) { aph::set_error(__VA_ARGS__); return 2; }                                     \
  } while (0)

// launch-error check without synchronising
#define APH_LAUNCH_OK()                                                                         \
  do {                                                                                          \
    cudaError_t _e = cudaGetLastError();                                                        \
    if (_e != cudaSuccess) {                                                                    \
      aph::set_error("%s:%d kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return 1;                                                                                 \
    }                                                                                           \
    aph::count_launch();                                                                        \
  } while (0)

// SMs of the current device, queried once per device: sizes the persistent grids and the grid-stride launches
// (132 on an H100 SXM, 114 on an H100 PCIe). A failed query only affects grid sizes, never results: it falls back to 132.
inline int num_sms() {
  static std::atomic<int> cache[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  int n = cache[dev].load(std::memory_order_relaxed);
  if (n <= 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cache[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

// Programmatic dependent launch: a kernel calls pdl_trigger() first thing (its dependents may start being scheduled as SMs
// drain) and pdl_wait() before its first global-memory access (blocks until the preceding grid has completed and flushed).
// The prologue in between (barrier init, descriptor prefetch, index setup) overlaps the predecessor's tail.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

bool pdl_enabled();            // api.cu: APH_PDL=1 enables (off by default: no measured gain on top of the graph cache)

// cudaLaunchKernelEx wrapper: optional cluster width and the programmatic-serialization attribute
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cluster, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[2];
  int n = 0;
  if (cluster > 1) { at[n].id = cudaLaunchAttributeClusterDimension; at[n].val.clusterDim.x = cluster; at[n].val.clusterDim.y = 1; at[n].val.clusterDim.z = 1; ++n; }
  if (pdl_enabled()) { at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[n].val.programmaticStreamSerializationAllowed = 1; ++n; }
  cfg.attrs = at; cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }

}  // namespace aph
