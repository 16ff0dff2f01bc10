// Host-side staging for the HOST-pointer entry points (vfi_*_interpolate_host): pageable caller memory <-> a small
// ring of pinned buffers <-> the GPU, so that a ComfyUI IMAGE tensor (pageable) moves at PCIe rate without pinning the
// caller's clip (the reference's loop does blocking `.to(device)` / `.cpu()` per batch, rife/__init__.py:195-207).
//   * CopyPool: a few persistent threads that split one large memcpy (one thread copies ~10 GB/s; PCIe Gen5 needs ~45).
//   * PinnedBuf: a cudaHostAlloc'ed buffer that is kept by the context and only ever grows.
// Plain C++ (no CUDA kernels); the pipelines themselves live next to their models (rife46.cu).
#pragma once
#include <cuda_runtime.h>

#include <condition_variable>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>
#if defined(__AVX2__)
#include <immintrin.h>
#endif

namespace vfi {

// Large host copy with non-temporal stores: the destination (a pinned staging slot or the output clip) is not read by
// the CPU again, so the lines are written without first being fetched (no read-for-ownership: a third less DRAM
// traffic than a cached copy) and without evicting the source stream from the cache.  Falls back to memcpy for small or
// unaligned-tail pieces and when the translation unit is built without AVX2.
inline bool use_stream_stores() {  // VFI_NT_COPY=0: plain memcpy (A/B runs)
  static const bool on = [] {
    const char* e = std::getenv("VFI_NT_COPY");
    return !(e && e[0] == '0');
  }();
  return on;
}

inline void stream_copy(void* dst, const void* src, size_t bytes) {
#if defined(__AVX2__)
  if (bytes >= (256u << 10) && use_stream_stores()) {
    uint8_t* d = static_cast<uint8_t*>(dst);
    const uint8_t* s = static_cast<const uint8_t*>(src);
    const size_t head = (32 - (reinterpret_cast<uintptr_t>(d) & 31)) & 31;
    if (head) {
      std::memcpy(d, s, head);
      d += head;
      s += head;
      bytes -= head;
    }
    const size_t blocks = bytes / 128;
    for (size_t i = 0; i < blocks; ++i) {
      const __m256i a = _mm256_loadu_si256(reinterpret_cast<const __m256i*>(s));
      const __m256i b = _mm256_loadu_si256(reinterpret_cast<const __m256i*>(s + 32));
      const __m256i c = _mm256_loadu_si256(reinterpret_cast<const __m256i*>(s + 64));
      const __m256i e = _mm256_loadu_si256(reinterpret_cast<const __m256i*>(s + 96));
      _mm256_stream_si256(reinterpret_cast<__m256i*>(d), a);
      _mm256_stream_si256(reinterpret_cast<__m256i*>(d + 32), b);
      _mm256_stream_si256(reinterpret_cast<__m256i*>(d + 64), c);
      _mm256_stream_si256(reinterpret_cast<__m256i*>(d + 96), e);
      s += 128;
      d += 128;
    }
    _mm_sfence();
    bytes -= blocks * 128;
    if (bytes) std::memcpy(d, s, bytes);
    return;
  }
#endif
  std::memcpy(dst, src, bytes);
}

class CopyPool {
 public:
  explicit CopyPool(int nthreads) {
    if (nthreads < 1) nthreads = 1;
    for (int i = 0; i < nthreads; ++i) workers_.emplace_back([this, i, nthreads] { run(i, nthreads); });
  }
  ~CopyPool() {
    {
      std::lock_guard<std::mutex> l(m_);
      stop_ = true;
      ++gen_;
    }
    cv_.notify_all();
    for (auto& t : workers_) t.join();
  }
  CopyPool(const CopyPool&) = delete;
  CopyPool& operator=(const CopyPool&) = delete;

  // blocking; one caller at a time (each pipeline thread owns its pool)
  void copy(void* dst, const void* src, size_t bytes) {
    if (bytes < (1u << 20) || workers_.size() == 1) {  // not worth a hand-off
      std::memcpy(dst, src, bytes);
      return;
    }
    dispatch(dst, src, bytes, 0);
  }
  // dst[i*3 + k] = src[i*C + k], k < 3, for `px` fp32 pixels: the first three channels of an NHWC frame (C == 3: memcpy)
  void copy_rgb(float* dst, const float* src, size_t px, int C) {
    if (C == 3) {
      copy(dst, src, px * 3 * sizeof(float));
      return;
    }
    dispatch(dst, src, px, C);
  }

 private:
  void run(int idx, int n) {
    uint64_t seen = 0;
    for (;;) {
      uint8_t* d;
      const uint8_t* s;
      size_t bytes;
      int C;
      {
        std::unique_lock<std::mutex> l(m_);
        cv_.wait(l, [&] { return gen_ != seen; });
        seen = gen_;
        if (stop_) return;
        d = dst_;
        s = src_;
        bytes = bytes_;
        C = chan_;
      }
      if (C == 0) {
        // 4 KB-aligned chunk boundaries (whole pages per thread)
        const size_t chunk = ((bytes + n - 1) / n + 4095) & ~(size_t)4095;
        const size_t lo = std::min(bytes, chunk * idx), hi = std::min(bytes, chunk * (idx + 1));
        if (hi > lo) stream_copy(d + lo, s + lo, hi - lo);
      } else {  // `bytes` counts pixels here
        const size_t chunk = (bytes + n - 1) / n;
        const size_t lo = std::min(bytes, chunk * idx), hi = std::min(bytes, chunk * (idx + 1));
        float* df = reinterpret_cast<float*>(d);
        const float* sf = reinterpret_cast<const float*>(s);
        for (size_t i = lo; i < hi; ++i) {
          df[i * 3 + 0] = sf[i * C + 0];
          df[i * 3 + 1] = sf[i * C + 1];
          df[i * 3 + 2] = sf[i * C + 2];
        }
      }
      {
        std::lock_guard<std::mutex> l(m_);
        if (--pending_ == 0) done_.notify_all();
      }
    }
  }
  void dispatch(void* dst, const void* src, size_t n, int chan) {
    {
      std::lock_guard<std::mutex> l(m_);
      dst_ = static_cast<uint8_t*>(dst);
      src_ = static_cast<const uint8_t*>(src);
      bytes_ = n;
      chan_ = chan;
      pending_ = (int)workers_.size();
      ++gen_;
    }
    cv_.notify_all();
    std::unique_lock<std::mutex> l(m_);
    done_.wait(l, [this] { return pending_ == 0; });
  }
  std::vector<std::thread> workers_;
  std::mutex m_;
  std::condition_variable cv_, done_;
  uint64_t gen_ = 0;
  bool stop_ = false;
  uint8_t* dst_ = nullptr;
  const uint8_t* src_ = nullptr;
  size_t bytes_ = 0;
  int chan_ = 0;  // 0: byte copy; C > 3: first-three-channels copy of `bytes_` pixels
  int pending_ = 0;
};

struct PinnedBuf {
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t ensure(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    release();
    cudaError_t e = cudaHostAlloc(&p, bytes, cudaHostAllocDefault);
    if (e == cudaSuccess) cap = bytes;
    return e;
  }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
  }
};

// true when `ptr` is page-locked memory CUDA knows (cudaHostAlloc / cudaHostRegister / torch pin_memory)
inline bool is_pinned_host(const void* ptr) {
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeHost;
}

inline int env_int(const char* name, int dflt, int lo, int hi) {
  const char* e = std::getenv(name);
  if (!e || !*e) return dflt;
  const int v = std::atoi(e);
  return v < lo ? lo : (v > hi ? hi : v);
}

}  // namespace vfi
