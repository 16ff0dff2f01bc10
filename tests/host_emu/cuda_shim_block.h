// Host emulation with the FULL launch geometry (TEST INFRASTRUCTURE): every block of a launch runs through
// block_emu::run_block (one fiber per thread, __syncthreads() = yield), blocks in turn.  For kernels that index with
// blockIdx.{x,y,z} / threadIdx.x directly instead of a grid-stride loop (csrc/elementwise.cu) and for the few with
// cooperative shared-memory loads.  Plus the CUDA runtime calls csrc/rife46.cu makes, as host stubs (one "device",
// synchronous "streams").
#pragma once
#define VFI_HOST_EMU 1
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <cstring>

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#undef __global__
#undef __device__
#undef __host__
#undef __forceinline__
#undef __shared__
#undef __restrict__
#include "block_emu.h"
#define __device__
#define __host__
#define __forceinline__ inline
#define __grid_constant__
#define __launch_bounds__(...)
using std::isfinite;
using std::max;
using std::min;
template <typename T>
static inline T __ldg(const T* p) { return *p; }
#include <atomic>
template <typename F>
static inline F atomicAdd(F* p, F v) {  // float / double; blocks run on several host threads
  std::atomic_ref<F> a(*p);
  F o = a.load();
  while (!a.compare_exchange_weak(o, o + v)) {
  }
  return o;
}

static inline float4 atomicAdd(float4* p, float4 v) {  // the 16-byte vector atomic of sm_90+: four scalar atomics here
  float4 o;
  o.x = atomicAdd(&p->x, v.x);
  o.y = atomicAdd(&p->y, v.y);
  o.z = atomicAdd(&p->z, v.z);
  o.w = atomicAdd(&p->w, v.w);
  return o;
}
// warp shuffle through a per-block exchange buffer: every thread of the block calls it (the kernels that shuffle do so
// uniformly), the two block barriers stand in for the lock-step of a warp
static thread_local float emu_shfl_buf[1024];
static inline float __shfl_xor_sync(unsigned, float v, int lane_mask) {
  emu_shfl_buf[threadIdx.x] = v;
  __syncthreads();
  const float r = emu_shfl_buf[threadIdx.x ^ (unsigned)lane_mask];
  __syncthreads();
  return r;
}

#define VFI_DYN_SMEM(type, name) type* name = reinterpret_cast<type*>(emu_dyn_smem)
// blocks are dealt round-robin to up to 16 host threads; inside a block the threads are fibers (block_emu.h)
#include <thread>
#include <vector>
#define VFI_LAUNCH(kernel, grid, block, smem, stream, ...)                                          \
  do {                                                                                               \
    const dim3 _g(grid), _b(block);                                                                  \
    const size_t _nb = (size_t)_g.x * _g.y * _g.z;                                                   \
    unsigned _t = std::thread::hardware_concurrency();                                               \
    _t = _t < 1 ? 1 : (_t > 16 ? 16 : _t);                                                           \
    if ((size_t)_t > _nb) _t = (unsigned)_nb;                                                        \
    auto _work = [&](unsigned _w) {                                                                  \
      std::vector<char> _dyn((size_t)(smem) + 64);                                                   \
      emu_dyn_smem = _dyn.data();                                                                    \
      gridDim.x = _g.x; gridDim.y = _g.y; gridDim.z = _g.z;                                          \
      blockDim.x = _b.x; blockDim.y = 1; blockDim.z = 1;                                             \
      for (size_t _i = _w; _i < _nb; _i += _t) {                                                     \
        blockIdx.x = (unsigned)(_i % _g.x);                                                          \
        blockIdx.y = (unsigned)((_i / _g.x) % _g.y);                                                 \
        blockIdx.z = (unsigned)(_i / ((size_t)_g.x * _g.y));                                         \
        block_emu::run_block((int)_b.x, [&]() { kernel(__VA_ARGS__); });                             \
      }                                                                                              \
    };                                                                                               \
    if (_t <= 1) {                                                                                   \
      _work(0);                                                                                      \
    } else {                                                                                         \
      std::vector<std::thread> _th;                                                                  \
      for (unsigned _w = 0; _w < _t; ++_w) _th.emplace_back(_work, _w);                              \
      for (auto& _h : _th) _h.join();                                                                \
    }                                                                                                \
  } while (0)

static inline cudaError_t emu_malloc(void** p, size_t n) {
  const size_t bytes = ((n ? n : 1) + 255) / 256 * 256;
  *p = std::aligned_alloc(256, bytes);
  if (*p) std::memset(*p, 0, bytes);
  return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
static inline cudaError_t emu_props(cudaDeviceProp* p, int) {
  std::memset(p, 0, sizeof(*p));
  p->major = 9;
  p->multiProcessorCount = 132;
  return cudaSuccess;
}
static inline cudaError_t emu_memcpy(void* d, const void* s, size_t n) {
  std::memcpy(d, s, n);
  return cudaSuccess;
}
#define cudaMalloc(p, n) emu_malloc((void**)(p), (n))
#define cudaFree(p) (std::free(p), cudaSuccess)
#define cudaMemcpy(d, s, n, k) emu_memcpy((d), (s), (n))
#define cudaMemcpyAsync(d, s, n, k, st) emu_memcpy((d), (s), (n))
#define cudaMemsetAsync(d, v, n, st) (std::memset((d), (v), (n)), cudaSuccess)
#define cudaSetDevice(d) cudaSuccess
#define cudaGetLastError() cudaSuccess
#define cudaGetErrorString(e) "emulated CUDA error"
#define cudaGetDeviceCount(p) (*(p) = 1, cudaSuccess)
#define cudaGetDeviceProperties(p, d) emu_props((p), (d))
#define cudaDeviceSynchronize() cudaSuccess
#define cudaStreamSynchronize(s) cudaSuccess
#define cudaGetDevice(p) (*(p) = 0, cudaSuccess)
#define cudaDeviceGetAttribute(v, a, d) (*(v) = 132, cudaSuccess)
#define cudaStreamCreateWithFlags(p, f) (*(p) = nullptr, cudaSuccess)
#define cudaStreamDestroy(s) cudaSuccess
#define cudaStreamWaitEvent(s, e, f) cudaSuccess
#define cudaEventCreateWithFlags(p, f) (*(p) = nullptr, cudaSuccess)
#define cudaEventRecord(e, s) cudaSuccess
#define cudaEventDestroy(e) cudaSuccess
#define cudaFuncSetAttribute(k, a, v) cudaSuccess
// the host-pointer pipeline's staging (csrc/hoststage.h): every caller buffer counts as pageable here, so the emulation
// exercises the pinned-ring / uploader / downloader threads
#define cudaEventSynchronize(e) cudaSuccess
#define cudaEventCreate(p) (*(p) = nullptr, cudaSuccess)
#define cudaEventElapsedTime(ms, a, b) (*(ms) = 0.f, cudaSuccess)
#define cudaHostAlloc(p, n, f) emu_malloc((void**)(p), (n))
#define cudaFreeHost(p) (std::free(p), cudaSuccess)
#define cudaPointerGetAttributes(a, p) ((a)->type = cudaMemoryTypeUnregistered, cudaSuccess)
