// HBM-bound kernels of the Sepconv trunk (vfi_models/sepconv/sepconv_enhanced.py, Network.forward :605-706): everything
// that is not a >= 64-channel conv or the separable-kernel op itself.  16-bit activations are dense NHWC tensors.
//
//   sep_stats       sum / sum of squares of the (replicate-padded-to-even) pair        :622-633 (mean, unbiased std)
//                   per-block partials, then summed in a fixed order: the same call gives the same bits
//   sep_input_conv  (x - mean) / (std + 1e-7) -> Conv2d(3,16,3,pad 1) per frame, cat -> PReLU -> space-to-depth
//                   = the input of the first stride-2 conv                             :544-547, :640-642, :553
//   prelu_s2d16     PReLU + space-to-depth (zero filled past an odd edge): input of a stride-2 conv   :110-131
//   prelu16         PReLU                                                               :186-193
//   prelu_up2_16    PReLU (slope 1 = none) -> bilinear x2 (scale_factor 2, align_corners=False) -> crop to the finer
//                   level's size                                                        :150-156, :479-496
//   add_crop16      x[B,H,W,C] += v[B,Hv,Wv,C][:, :H, :W]  (Hv >= H, Wv >= W)                :479-496
//   sep_coeff_nchw  head output [B,H,W,64] 16-bit -> [B,51,H,W] fp32 (the op's layout)   :683-686
//   sep_pad_input   frame -> [B,4,He+50,We+50] fp32: replicate padding (to even, then by 25) + a channel of ones  :644-681
//   sep_finish      (o1 + o2)[:3] / normaliser (|n| < 0.01 -> 1), crop, NHWC             :688-702
#include "ptx.cuh"
#include "vfi_internal.h"

namespace vfi {

namespace {

template <typename T>
struct V8 {
  uint4 u;
  __device__ __forceinline__ void unpack(float (&f)[8]) const {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 p = Pack2<T>::unpack(w[i]);
      f[2 * i] = p.x;
      f[2 * i + 1] = p.y;
    }
  }
  __device__ __forceinline__ void pack(const float (&f)[8]) {
    u.x = Pack2<T>::pack(f[0], f[1]);
    u.y = Pack2<T>::pack(f[2], f[3]);
    u.z = Pack2<T>::pack(f[4], f[5]);
    u.w = Pack2<T>::pack(f[6], f[7]);
  }
};

inline int sgrid(size_t total, int threads) {
  size_t b = (total + threads - 1) / threads;
  return (int)(b < 1 ? 1 : (b > 1048576 ? 1048576 : b));
}

__device__ __forceinline__ float prelu(float v, float s) { return v > 0.f ? v : s * v; }

// ---- statistics of the padded pair: stats[2*b] = sum, stats[2*b+1] = sum of squares (double), over 2 frames x 3 x He x We.
// Block (x, b) writes its partial sums to partial[b][x]; sep_stats_sum_kernel adds them in index order (double atomics
// across blocks would add them in whatever order the blocks finish, and the last bits would differ from call to call).
__global__ void sep_stats_kernel(const float* __restrict__ frames, int cstride, SepPairIdx idx, int H, int W, int He, int We,
                                 double* __restrict__ partial) {
  const int b = blockIdx.y;
  const size_t per = (size_t)He * We;
  double s = 0.0, q = 0.0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < 2 * per; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i / per);
    const size_t px = i - (size_t)k * per;
    const int y = min((int)(px / We), H - 1), x = min((int)(px % We), W - 1);  // replicate pad to even (:611-618)
    const float* p = frames + (((size_t)(k ? idx.f1[b] : idx.f0[b]) * H + y) * W + x) * cstride;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double v = (double)p[c];
      s += v;
      q += v * v;
    }
  }
  __shared__ double sh[2][256];
  sh[0][threadIdx.x] = s;
  sh[1][threadIdx.x] = q;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) {
      sh[0][threadIdx.x] += sh[0][threadIdx.x + o];
      sh[1][threadIdx.x] += sh[1][threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    double* p = partial + 2 * ((size_t)b * gridDim.x + blockIdx.x);
    p[0] = sh[0][0];
    p[1] = sh[1][0];
  }
}

// one block per pair: stats[2*b], stats[2*b+1] = the sums of partial[b][0..nblk), in a fixed order
__global__ void sep_stats_sum_kernel(const double* __restrict__ partial, int nblk, double* __restrict__ stats) {
  const int b = blockIdx.x;
  double s = 0.0, q = 0.0;
  for (int i = threadIdx.x; i < nblk; i += blockDim.x) {
    s += partial[2 * ((size_t)b * nblk + i)];
    q += partial[2 * ((size_t)b * nblk + i) + 1];
  }
  __shared__ double sh[2][256];
  sh[0][threadIdx.x] = s;
  sh[1][threadIdx.x] = q;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) {
      sh[0][threadIdx.x] += sh[0][threadIdx.x + o];
      sh[1][threadIdx.x] += sh[1][threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    stats[2 * b] = sh[0][0];
    stats[2 * b + 1] = sh[1][0];
  }
}

// ---- netInput on both normalised frames + PReLU + space-to-depth: out [B, He/2, We/2, (a, b, 32)] 16-bit, channel
// = frame * 16 + c.  Two threads per pixel (one per frame).  Zero padding applies to the NORMALISED image (:544-547).
template <typename T>
__global__ void sep_input_conv_kernel(const float* __restrict__ frames, int cstride, SepPairIdx idx, int H, int W, int He,
                                      int We, const double* __restrict__ stats, const float* __restrict__ w,
                                      const float* __restrict__ bias, float slope, T* __restrict__ out, int B) {
  __shared__ float ws[27 * 16];
  __shared__ float bs[16];
  for (int i = threadIdx.x; i < 27 * 16; i += blockDim.x) {
    const int k = i / 16, o = i - k * 16;
    ws[i] = w[o * 27 + k];
  }
  for (int i = threadIdx.x; i < 16; i += blockDim.x) bs[i] = bias[i];
  __syncthreads();
  const size_t per = (size_t)He * We;
  const size_t total = (size_t)B * per * 2;
  const double cnt = 2.0 * 3.0 * (double)per;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i & 1);
    const size_t pi = i >> 1;
    const int b = (int)(pi / per);
    const size_t px = pi - (size_t)b * per;
    const int y = (int)(px / We), x = (int)(px % We);
    const double mean_d = stats[2 * b] / cnt;
    const double var_d = (stats[2 * b + 1] - cnt * mean_d * mean_d) / (cnt - 1.0);  // torch.std: unbiased (:630)
    const float mean = (float)mean_d;
    const float inv = 1.f / ((float)sqrt(var_d > 0.0 ? var_d : 0.0) + 0.0000001f);
    const float* img = frames + (size_t)(k ? idx.f1[b] : idx.f0[b]) * H * W * cstride;
    float v[27];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int yy = y + ky - 1, xx = x + kx - 1;
        const bool ok = yy >= 0 && yy < He && xx >= 0 && xx < We;
        const float* s = img + ((size_t)min(max(yy, 0), H - 1) * W + min(max(xx, 0), W - 1)) * cstride;
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c * 9 + ky * 3 + kx] = ok ? (s[c] - mean) * inv : 0.f;
      }
    float acc[16];
#pragma unroll
    for (int o = 0; o < 16; ++o) acc[o] = bs[o];
#pragma unroll
    for (int t = 0; t < 27; ++t)
#pragma unroll
      for (int o = 0; o < 16; ++o) acc[o] = fmaf(v[t], ws[t * 16 + o], acc[o]);
    float f0[8], f1[8];
#pragma unroll
    for (int o = 0; o < 8; ++o) {
      f0[o] = prelu(acc[o], slope);
      f1[o] = prelu(acc[8 + o], slope);
    }
    V8<T> p0, p1;
    p0.pack(f0);
    p1.pack(f1);
    T* d = out + ((((size_t)b * (He >> 1) + (y >> 1)) * (We >> 1) + (x >> 1)) * 128 + ((y & 1) * 2 + (x & 1)) * 32 + k * 16);
    *reinterpret_cast<uint4*>(d) = p0.u;
    *reinterpret_cast<uint4*>(d + 8) = p1.u;
  }
}

// ---- x [B,H,W,C] -> [B, ceil(H/2), ceil(W/2), (a, b, C)] with PReLU; cells past an odd edge are zero (= the conv's padding)
template <typename T>
__global__ void prelu_s2d16_kernel(const T* __restrict__ in, T* __restrict__ out, float slope, int C8, int B, int H, int W) {
  const int Ho = (H + 1) >> 1, Wo = (W + 1) >> 1;
  const size_t total = (size_t)B * Ho * Wo * 4 * C8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C8);
    size_t r = i / C8;
    const int ab = (int)(r & 3);
    r >>= 2;
    const int x = (int)(r % Wo);
    const int y = (int)((r / Wo) % Ho);
    const int b = (int)(r / ((size_t)Wo * Ho));
    const int sy = 2 * y + (ab >> 1), sx = 2 * x + (ab & 1);
    V8<T> v;
    v.u = make_uint4(0u, 0u, 0u, 0u);
    if (sy < H && sx < W) {
      v.u = *reinterpret_cast<const uint4*>(in + ((((size_t)b * H + sy) * W + sx) * C8 + c) * 8);
      float f[8];
      v.unpack(f);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = prelu(f[j], slope);
      v.pack(f);
    }
    *reinterpret_cast<uint4*>(out + i * 8) = v.u;
  }
}

template <typename T>
__global__ void prelu16_kernel(const T* __restrict__ in, T* __restrict__ out, float slope, size_t n8) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (size_t)gridDim.x * blockDim.x) {
    V8<T> v;
    v.u = *reinterpret_cast<const uint4*>(in + i * 8);
    float f[8];
    v.unpack(f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = prelu(f[j], slope);
    v.pack(f);
    *reinterpret_cast<uint4*>(out + i * 8) = v.u;
  }
}

// ---- out[B,Ht,Wt,C] = crop(interpolate(prelu(in [B,h,w,C]), scale_factor=2, bilinear)), Ht <= 2h, Wt <= 2w.
// ATen with a scale factor: src = max((dst + 0.5) * 0.5 - 0.5, 0), second tap clamped.
template <typename T>
__global__ void prelu_up2_16_kernel(const T* __restrict__ in, T* __restrict__ out, float slope, int C8, int B, int h, int w,
                                    int Ht, int Wt) {
  const size_t total = (size_t)B * Ht * Wt * C8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C8);
    size_t r = i / C8;
    const int x = (int)(r % Wt);
    const int y = (int)((r / Wt) % Ht);
    const int b = (int)(r / ((size_t)Wt * Ht));
    const float fy = fmaxf(((float)y + 0.5f) * 0.5f - 0.5f, 0.f), fx = fmaxf(((float)x + 0.5f) * 0.5f - 0.5f, 0.f);
    const int y0 = min((int)fy, h - 1), x0 = min((int)fx, w - 1);
    const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
    const float ly = fy - (float)y0, lx = fx - (float)x0;
    const T* base = in + (size_t)b * h * w * C8 * 8 + c * 8;
    float a[8], o[8];
    V8<T> v;
    const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx), w11 = ly * lx;
    v.u = *reinterpret_cast<const uint4*>(base + ((size_t)y0 * w + x0) * C8 * 8);
    v.unpack(a);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = prelu(a[j], slope) * w00;
    v.u = *reinterpret_cast<const uint4*>(base + ((size_t)y0 * w + x1) * C8 * 8);
    v.unpack(a);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = fmaf(prelu(a[j], slope), w01, o[j]);
    v.u = *reinterpret_cast<const uint4*>(base + ((size_t)y1 * w + x0) * C8 * 8);
    v.unpack(a);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = fmaf(prelu(a[j], slope), w10, o[j]);
    v.u = *reinterpret_cast<const uint4*>(base + ((size_t)y1 * w + x1) * C8 * 8);
    v.unpack(a);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = fmaf(prelu(a[j], slope), w11, o[j]);
    v.pack(o);
    *reinterpret_cast<uint4*>(out + i * 8) = v.u;
  }
}

template <typename T>
__global__ void add_crop16_kernel(const T* __restrict__ v, int Hv, int Wv, T* __restrict__ x, int C8, int B, int H, int W) {
  const size_t total = (size_t)B * H * W * C8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C8);
    size_t r = i / C8;
    const int xx = (int)(r % W);
    const int y = (int)((r / W) % H);
    const int b = (int)(r / ((size_t)W * H));
    V8<T> a, d;
    a.u = *reinterpret_cast<const uint4*>(x + i * 8);
    d.u = *reinterpret_cast<const uint4*>(v + ((((size_t)b * Hv + y) * Wv + xx) * C8 + c) * 8);
    float fa[8], fd[8];
    a.unpack(fa);
    d.unpack(fd);
#pragma unroll
    for (int j = 0; j < 8; ++j) fa[j] += fd[j];
    a.pack(fa);
    *reinterpret_cast<uint4*>(x + i * 8) = a.u;
  }
}

// [B, HW, pitch] 16-bit (pitch = 64: the head's padded channel count) -> [B, K, HW] fp32.  Tiles of 32 pixels through shared
// memory so that both sides are coalesced: a pixel's channels are read as 32-bit words (128 B per pixel), a channel's 32 pixels
// are written as 128 B (one thread per output element would read a 2-byte value with a 128-byte stride).
// Written for any blockDim (the host emulation runs it with one thread per block).
template <typename T>
__global__ void sep_coeff_nchw_kernel(const T* __restrict__ in, int pitch, float* __restrict__ out, int K, int B, size_t hw) {
  __shared__ float tile[64][33];
  const uint32_t* in32 = reinterpret_cast<const uint32_t*>(in);
  const int wpp = pitch >> 1;                         // 32-bit words per pixel
  const int kw = (K + 1) >> 1;                        // words that hold the K channels
  const size_t tiles_per_img = (hw + 31) / 32;
  const size_t ntiles = (size_t)B * tiles_per_img;
  for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int b = (int)(t / tiles_per_img);
    const size_t p0 = (t % tiles_per_img) * 32;
    for (int e = threadIdx.x; e < 32 * kw; e += blockDim.x) {
      const int p = e / kw, wq = e - p * kw;
      if (p0 + p < hw) {
        const float2 v = Pack2<T>::unpack(in32[((size_t)b * hw + p0 + p) * wpp + wq]);
        tile[2 * wq][p] = v.x;
        tile[2 * wq + 1][p] = v.y;
      }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < 32 * K; e += blockDim.x) {
      const int k = e >> 5, p = e & 31;
      if (p0 + p < hw) out[((size_t)b * K + k) * hw + p0 + p] = tile[k][p];
    }
    __syncthreads();
  }
}

__global__ void sep_pad_input_kernel(const float* __restrict__ frames, int cstride, SepPairIdx idx, int which, int H, int W,
                                     int Hp, int Wp, float* __restrict__ out, int B) {
  const size_t per = (size_t)Hp * Wp;
  const size_t total = (size_t)B * 4 * per;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t px = i % per;
    const int c = (int)((i / per) & 3);
    const int b = (int)(i / (4 * per));
    const int y = min(max((int)(px / Wp) - 25, 0), H - 1), x = min(max((int)(px % Wp) - 25, 0), W - 1);
    const int f = which ? idx.f1[b] : idx.f0[b];
    out[i] = c == 3 ? 1.f : frames[(((size_t)f * H + y) * W + x) * cstride + c];
  }
}

__global__ void sep_finish_kernel(const float* __restrict__ o1, const float* __restrict__ o2, float* __restrict__ out, int B,
                                  int H, int W, int He, int We) {
  const size_t total = (size_t)B * H * W;
  const size_t pe = (size_t)He * We;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const int y = (int)((i / W) % H);
    const int b = (int)(i / ((size_t)W * H));
    const size_t base = (size_t)b * 4 * pe + (size_t)y * We + x;
    float n = o1[base + 3 * pe] + o2[base + 3 * pe];
    if (fabsf(n) < 0.01f) n = 1.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) out[i * 3 + c] = (o1[base + c * pe] + o2[base + c * pe]) / n;
  }
}

}  // namespace

int sep_stats_blocks(int He, int We) { return sgrid((size_t)2 * He * We, 256 * 8); }

cudaError_t launch_sep_stats(const float* frames, int cstride, const SepPairIdx& idx, int B, int H, int W, int He, int We,
                             double* stats, double* partial, cudaStream_t st) {
  const int nb = sep_stats_blocks(He, We);
  VFI_LAUNCH(sep_stats_kernel, dim3((unsigned)nb, (unsigned)B), 256, 0, st, frames, cstride, idx, H, W, He, We, partial);
  VFI_LAUNCH(sep_stats_sum_kernel, B, 256, 0, st, partial, nb, stats);
  return cudaGetLastError();
}

cudaError_t launch_sep_input_conv(int op, const float* frames, int cstride, const SepPairIdx& idx, int B, int H, int W, int He,
                                  int We, const double* stats, const float* w, const float* bias, float slope, void* out,
                                  cudaStream_t st) {
  const int g = sgrid((size_t)B * He * We * 2, 128);
  if (op == OP_BF16)
    VFI_LAUNCH(sep_input_conv_kernel<__nv_bfloat16>, g, 128, 0, st, frames, cstride, idx, H, W, He, We, stats, w, bias, slope,
                                                            (__nv_bfloat16*)out, B);
  else
    VFI_LAUNCH(sep_input_conv_kernel<__half>, g, 128, 0, st, frames, cstride, idx, H, W, He, We, stats, w, bias, slope, (__half*)out, B);
  return cudaGetLastError();
}

cudaError_t launch_prelu_s2d16(int op, const void* in, void* out, float slope, int C, int B, int H, int W, cudaStream_t st) {
  if (C & 7) return cudaErrorInvalidValue;
  const int g = sgrid((size_t)B * ((H + 1) / 2) * ((W + 1) / 2) * 4 * (C / 8), 256);
  if (op == OP_BF16)
    VFI_LAUNCH(prelu_s2d16_kernel<__nv_bfloat16>, g, 256, 0, st, (const __nv_bfloat16*)in, (__nv_bfloat16*)out, slope, C / 8, B, H, W);
  else
    VFI_LAUNCH(prelu_s2d16_kernel<__half>, g, 256, 0, st, (const __half*)in, (__half*)out, slope, C / 8, B, H, W);
  return cudaGetLastError();
}

cudaError_t launch_prelu16(int op, const void* in, void* out, float slope, size_t n, cudaStream_t st) {
  if (n & 7) return cudaErrorInvalidValue;
  const int g = sgrid(n / 8, 256);
  if (op == OP_BF16)
    VFI_LAUNCH(prelu16_kernel<__nv_bfloat16>, g, 256, 0, st, (const __nv_bfloat16*)in, (__nv_bfloat16*)out, slope, n / 8);
  else
    VFI_LAUNCH(prelu16_kernel<__half>, g, 256, 0, st, (const __half*)in, (__half*)out, slope, n / 8);
  return cudaGetLastError();
}

cudaError_t launch_prelu_up2_16(int op, const void* in, void* out, float slope, int C, int B, int h, int w, int Ht, int Wt,
                                cudaStream_t st) {
  if ((C & 7) || Ht > 2 * h || Wt > 2 * w) return cudaErrorInvalidValue;
  const int g = sgrid((size_t)B * Ht * Wt * (C / 8), 256);
  if (op == OP_BF16)
    VFI_LAUNCH(prelu_up2_16_kernel<__nv_bfloat16>, g, 256, 0, st, (const __nv_bfloat16*)in, (__nv_bfloat16*)out, slope, C / 8, B, h, w,
                                                          Ht, Wt);
  else
    VFI_LAUNCH(prelu_up2_16_kernel<__half>, g, 256, 0, st, (const __half*)in, (__half*)out, slope, C / 8, B, h, w, Ht, Wt);
  return cudaGetLastError();
}

cudaError_t launch_add_crop16(int op, const void* v, int Hv, int Wv, void* x, int C, int B, int H, int W, cudaStream_t st) {
  if ((C & 7) || Hv < H || Wv < W) return cudaErrorInvalidValue;
  const int g = sgrid((size_t)B * H * W * (C / 8), 256);
  if (op == OP_BF16)
    VFI_LAUNCH(add_crop16_kernel<__nv_bfloat16>, g, 256, 0, st, (const __nv_bfloat16*)v, Hv, Wv, (__nv_bfloat16*)x, C / 8, B, H, W);
  else
    VFI_LAUNCH(add_crop16_kernel<__half>, g, 256, 0, st, (const __half*)v, Hv, Wv, (__half*)x, C / 8, B, H, W);
  return cudaGetLastError();
}

cudaError_t launch_sep_coeff_nchw(int op, const void* in, int pitch, float* out, int K, int B, int H, int W, cudaStream_t st) {
  const size_t hw = (size_t)H * W;
  if (K > 64 || (pitch & 1) || K > pitch) return cudaErrorInvalidValue;
  const int g = sgrid((size_t)B * ((hw + 31) / 32) * 256, 256);  // one block per tile of 32 pixels (capped, grid-stride)
  if (op == OP_BF16)
    VFI_LAUNCH(sep_coeff_nchw_kernel<__nv_bfloat16>, g, 256, 0, st, (const __nv_bfloat16*)in, pitch, out, K, B, hw);
  else
    VFI_LAUNCH(sep_coeff_nchw_kernel<__half>, g, 256, 0, st, (const __half*)in, pitch, out, K, B, hw);
  return cudaGetLastError();
}

cudaError_t launch_sep_pad_input(const float* frames, int cstride, const SepPairIdx& idx, int which, int B, int H, int W,
                                 int Hp, int Wp, float* out, cudaStream_t st) {
  VFI_LAUNCH(sep_pad_input_kernel, sgrid((size_t)B * 4 * Hp * Wp, 256), 256, 0, st, frames, cstride, idx, which, H, W, Hp, Wp, out, B);
  return cudaGetLastError();
}

cudaError_t launch_sep_finish(const float* o1, const float* o2, float* out, int B, int H, int W, int He, int We,
                              cudaStream_t st) {
  VFI_LAUNCH(sep_finish_kernel, sgrid((size_t)B * H * W, 256), 256, 0, st, o1, o2, out, B, H, W, He, We);
  return cudaGetLastError();
}

}  // namespace vfi
