// Host emulation shim (TEST INFRASTRUCTURE): lets g++ compile the element-wise CUDA kernels of csrc/sepconv_elem.cu as plain
// C++ so that tests/test_sepconv_elem_host.py can run them on the CPU (one "thread", grid-stride loops cover everything)
// against numpy / torch restatements.  The tensor-core kernels are not emulated.  Never part of the product build.
#pragma once
#define VFI_HOST_EMU 1
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#undef __global__
#undef __device__
#undef __host__
#undef __forceinline__
#undef __shared__
#undef __restrict__
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __shared__ static thread_local
#define __restrict__
struct EmuDim {
  unsigned x = 0, y = 0, z = 0;
};
static thread_local EmuDim blockIdx, threadIdx;
static thread_local EmuDim blockDim{1, 1, 1}, gridDim{1, 1, 1};
static inline void __syncthreads() {}
#include <mutex>
static inline double atomicAdd(double* p, double v) {
  static std::mutex m;
  std::lock_guard<std::mutex> g(m);
  const double o = *p;
  *p += v;
  return o;
}
using std::max;
using std::min;

// ---- launches and the few runtime calls the schedules make, for the whole-path emulation (sepconv_full_emu.cpp)
#define __grid_constant__
// one host thread per emulated block in x (every kernel walks its range with a grid-stride loop), grid rows in turn
#include <thread>
#include <vector>
#define VFI_LAUNCH(kernel, grid, block, smem, stream, ...)                        \
  do {                                                                            \
    const dim3 _g(grid);                                                          \
    unsigned _t = std::thread::hardware_concurrency();                            \
    _t = _t < 1 ? 1 : (_t > 16 ? 16 : _t);                                        \
    if (_t > _g.x) _t = _g.x;                                                     \
    for (unsigned _y = 0; _y < _g.y; ++_y) {                                      \
      std::vector<std::thread> _th;                                               \
      for (unsigned _x = 0; _x < _t; ++_x)                                        \
        _th.emplace_back([&, _x]() {                                              \
          blockIdx.x = _x;                                                        \
          blockIdx.y = _y;                                                        \
          gridDim.x = _t;                                                         \
          kernel(__VA_ARGS__);                                                    \
        });                                                                       \
      for (auto& _h : _th) _h.join();                                             \
    }                                                                             \
  } while (0)
#include <cstdlib>
#include <cstring>
static inline cudaError_t emu_malloc(void** p, size_t n) {
  const size_t bytes = ((n ? n : 1) + 255) / 256 * 256;   // cudaMalloc alignment
  *p = std::aligned_alloc(256, bytes);
  if (*p) std::memset(*p, 0, bytes);
  return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
static inline cudaError_t emu_free(void* p) {
  std::free(p);
  return cudaSuccess;
}
static inline cudaError_t emu_memcpy(void* d, const void* s, size_t n, cudaMemcpyKind) {
  std::memcpy(d, s, n);
  return cudaSuccess;
}
static inline cudaError_t emu_memset_async(void* d, int v, size_t n, cudaStream_t) {
  std::memset(d, v, n);
  return cudaSuccess;
}
#define cudaMalloc(p, n) emu_malloc((void**)(p), (n))
#define cudaFree(p) emu_free(p)
#define cudaMemcpy(d, s, n, k) emu_memcpy((d), (s), (n), (k))
#define cudaMemcpyAsync(d, s, n, k, st) emu_memcpy((d), (s), (n), (k))
#define cudaMemsetAsync(d, v, n, st) emu_memset_async((d), (v), (n), (st))
#define cudaSetDevice(d) cudaSuccess
#define cudaGetLastError() cudaSuccess
#define cudaGetErrorString(e) "emulated CUDA error"
#define cudaGetDevice(p) (*(p) = 0, cudaSuccess)
#define cudaDeviceGetAttribute(v, a, d) (*(v) = 132, cudaSuccess)
#define cudaStreamSynchronize(s) cudaSuccess
#define cudaDeviceSynchronize() cudaSuccess
