// aph_common.cuh -- shared helpers for libaphb200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <utility>
#include <vector>

#include "../../include/aphb200.h"

namespace aph {

typedef __nv_bfloat16 bf16;

void set_error(const char* fmt, ...);          // defined in api.cu (thread-local message)
extern std::atomic<long long> g_launches;      // kernels launched by this library
extern std::atomic<long long> g_device_bytes;  // device bytes held by DeviceAllocs, Scratch and StreamTemp

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

// Blocks of 256 threads for a grid-stride loop over n items: one per 256 items, at least one, at most `per_sm` per SM.
inline int stride_blocks(size_t n, int per_sm) {
  const size_t b = (n + 255) / 256, cap = (size_t)per_sm * num_sms();
  return (int)(b < 1 ? 1 : b < cap ? b : cap);
}

// Raises `kernel`'s dynamic shared-memory limit on the current device to at least `bytes`. It never lowers it: the limit belongs
// to the kernel, so a launch that needs less must not break a larger one of the same kernel (two FFT plans of different sizes).
// With `max_carveout` it also asks once for the largest shared-memory carveout. The limit is read once and then cached per
// (kernel, device), so a launch that needs no more than before makes no attribute call.
inline int smem_at_least(const void* kernel, size_t bytes, bool max_carveout = false) {
  struct Conf { int smem; bool carveout; };
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, Conf> confs;
  int dev = 0;
  APH_CUDA_OK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  auto it = confs.find({kernel, dev});
  if (it == confs.end()) {
    cudaFuncAttributes fa;
    APH_CUDA_OK(cudaFuncGetAttributes(&fa, kernel));
    it = confs.insert({{kernel, dev}, Conf{fa.maxDynamicSharedSizeBytes, false}}).first;
  }
  Conf& c = it->second;
  if ((int)bytes > c.smem) {
    APH_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    c.smem = (int)bytes;
  }
  if (max_carveout && !c.carveout) {
    APH_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    c.carveout = true;
  }
  return 0;
}

// The three owner types below are the only code that allocates or frees device memory; aph_device_bytes() is their sum.
struct NoCopy { NoCopy() = default; NoCopy(const NoCopy&) = delete; NoCopy& operator=(const NoCopy&) = delete; };

// Device memory of a handle or plan: every allocation lives as long as its owner.
struct DeviceAllocs : NoCopy {
  int64_t bytes = 0;           // every allocation below
  std::vector<void*> allocs;
  ~DeviceAllocs() { for (void* p : allocs) cudaFree(p); g_device_bytes -= bytes; }
  template <typename Tp>
  int alloc(Tp** p, size_t count) {
    APH_CUDA_OK(cudaMalloc((void**)p, count * sizeof(Tp)));
    allocs.push_back(*p);
    bytes += (int64_t)(count * sizeof(Tp));
    g_device_bytes += (int64_t)(count * sizeof(Tp));
    return 0;
  }
};

// Library-owned device scratch (it survives torch.cuda.empty_cache()) that grows on demand. Growing waits for `st` first: work
// already queued there may still use the old buffer. One held for the life of the process is `static Scratch& s = *new Scratch;`,
// never destroyed: a cudaFree from a static destructor would run after the CUDA runtime may have unloaded.
struct Scratch : NoCopy {
  float* p = nullptr;
  size_t bytes = 0;
  ~Scratch() { cudaFree(p); g_device_bytes -= bytes; }
  int grow(size_t need, cudaStream_t st) {
    if (need <= bytes) return 0;
    APH_CUDA_OK(cudaStreamSynchronize(st));
    if (p) cudaFree(p);
    g_device_bytes -= bytes;
    p = nullptr; bytes = 0;
    APH_CUDA_OK(cudaMalloc(&p, need));
    bytes = need;
    g_device_bytes += bytes;
    return 0;
  }
};

// A stream-ordered temporary: allocated on a stream, and freed on it behind the work queued there when it goes out of scope.
template <typename T>
struct StreamTemp : NoCopy {
  T* p = nullptr;
  size_t bytes = 0;
  cudaStream_t st = nullptr;
  ~StreamTemp() { if (p) cudaFreeAsync(p, st); g_device_bytes -= bytes; }
  int alloc(size_t count, cudaStream_t s) {
    st = s;
    APH_CUDA_OK(cudaMallocAsync((void**)&p, count * sizeof(T), st));
    bytes = count * sizeof(T);
    g_device_bytes += bytes;
    return 0;
  }
};

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
// dst[k] += the block's sum of v[k], k < N, in fp64: each warp sums by shuffles, thread 0 adds the warps in index order, and one
// atomicAdd per value. Every thread of the block must call it (it synchronises), and the block must have at most 256 threads:
// every caller is __launch_bounds__(256) and launched with 256.
template <int N>
__device__ __forceinline__ void block_atomic_add_d(const double (&v)[N], double* dst) {
  double w[N];
#pragma unroll
  for (int k = 0; k < N; ++k) w[k] = warp_sum_d(v[k]);
  __shared__ double red[N][8];
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < N; ++k) red[k][wid] = w[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t[N] = {};
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) {
#pragma unroll
      for (int k = 0; k < N; ++k) t[k] += red[k][i];
    }
#pragma unroll
    for (int k = 0; k < N; ++k) atomicAdd(&dst[k], t[k]);
  }
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }

// Row length of the encoder's patch-embedding operand (conv1 as a GEMM): the 3 p^2 pixels of a patch, zero-padded to a
// multiple of 128 (the K step of the forward GEMM, and the N tile of the data-gradient GEMM, whose N is this length).
// 3072 for p = 32 and 768 for p = 16 (no padding), 640 for p = 14 (52 zero columns).
__host__ __device__ constexpr int patch_k(int p) { return (3 * p * p + 127) / 128 * 128; }

}  // namespace aph
