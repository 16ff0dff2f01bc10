// The kernels of the FLAVR path (flavr.cu) around its tensor-core convolutions, on the CUDA cores.
// Activations are 16-bit [image][H][W][C] tensors, image = sample * T + plane (T = 4 planes per window, NTHWC); the
// input frames and the output are fp32 NHWC.  Reference: vfi_models/flavr/flavr_arch.py, resnet_3D.py.
//
//   frame_sums  per-(image, channel) sums over the replicate-padded frame      InputPadder.pad flavr_arch.py:208-209
//   prep        padded frame minus the window's mean as float4 planes          UNet_3D_3D.forward :171-172
//   stem        Conv3d(3, 64, (3,7,7), stride (1,2,2), pad (1,3,3)) + ReLU     BasicStem resnet_3D.py:42-50
//   chan_sums   per-(sample, channel) partial sums of a conv output           SEGating.pool (AdaptiveAvgPool3d(1))
//   gate        sigmoid(W . mean + b) per (sample, channel)                    SEGating.attn_layer
//   apply       x * g (+ residual) -> ReLU / LeakyReLU(0.2) -> 16-bit, optionally from the four phases of a transposed
//               conv (depth-to-space) and optionally also as the space-to-depth copy a stride-2 conv reads
//   outconv     ReflectionPad2d(3) + Conv2d(64, 3, 7) + mean, centred crop     UNet_3D_3D.outconv :161-164, :192-196
#include "ptx.cuh"
#include "vfi_internal.h"

namespace vfi {

namespace {

inline int fl_grid(size_t total, int threads) {
  size_t b = (total + threads - 1) / threads;
  return (int)(b < 1 ? 1 : (b > 1048576 ? 1048576 : b));
}

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

template <typename T>
__device__ __forceinline__ void ld8(const T* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 v = Pack2<T>::unpack(w[i]);
    f[2 * i] = v.x;
    f[2 * i + 1] = v.y;
  }
}

template <typename T>
__device__ __forceinline__ void st8(T* p, const float (&f)[8]) {
  uint4 u;
  u.x = Pack2<T>::pack(f[0], f[1]);
  u.y = Pack2<T>::pack(f[2], f[3]);
  u.z = Pack2<T>::pack(f[4], f[5]);
  u.w = Pack2<T>::pack(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// one block per image (grid-stride): sum of each RGB channel over the Hp x Wp replicate-padded frame
__global__ void frame_sums_kernel(const float* __restrict__ frames, int cstride, const FlavrFrameIdx idx, int n_img, int H,
                                  int W, int Hp, int Wp, int pt, int pl, float* __restrict__ sums) {
  __shared__ double red[3][256];
  for (int img = blockIdx.x; img < n_img; img += gridDim.x) {
    const float* f = frames + (size_t)idx.i[img] * H * W * cstride;
    double a[3] = {0.0, 0.0, 0.0};
    for (int p = threadIdx.x; p < Hp * Wp; p += blockDim.x) {
      const int y = clampi(p / Wp - pt, 0, H - 1), x = clampi(p % Wp - pl, 0, W - 1);
      const float* s = f + ((size_t)y * W + x) * cstride;
      a[0] += s[0];
      a[1] += s[1];
      a[2] += s[2];
    }
    for (int c = 0; c < 3; ++c) red[c][threadIdx.x] = a[c];
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
      if ((int)threadIdx.x < s)
        for (int c = 0; c < 3; ++c) red[c][threadIdx.x] += red[c][threadIdx.x + s];
      __syncthreads();
    }
    if (threadIdx.x == 0)
      for (int c = 0; c < 3; ++c) sums[img * 3 + c] = (float)red[c][0];
    __syncthreads();
  }
}

// mean of sample k, channel c over its T planes (the padded frames)
__device__ __forceinline__ float window_mean(const float* sums, int k, int c, int T, float inv_count) {
  float s = 0.f;
  for (int t = 0; t < T; ++t) s += sums[(k * T + t) * 3 + c];
  return s * inv_count;
}

__global__ void prep_kernel(const float* __restrict__ frames, int cstride, const FlavrFrameIdx idx, int n_img, int T, int H,
                            int W, int Hp, int Wp, int pt, int pl, const float* __restrict__ sums, float inv_count,
                            float4* __restrict__ out) {
  const size_t hw = (size_t)Hp * Wp, total = (size_t)n_img * hw;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int img = (int)(i / hw);
    const int p = (int)(i - (size_t)img * hw);
    const int y = clampi(p / Wp - pt, 0, H - 1), x = clampi(p % Wp - pl, 0, W - 1);
    const float* s = frames + (((size_t)idx.i[img] * H + y) * W + x) * cstride;
    const int k = img / T;
    out[i] = make_float4(s[0] - window_mean(sums, k, 0, T, inv_count), s[1] - window_mean(sums, k, 1, T, inv_count),
                         s[2] - window_mean(sums, k, 2, T, inv_count), 0.f);
  }
}

// stem: a thread computes four neighbouring output pixels of a row for 32 of the 64 output channels (which half is
// uniform over a warp, so the weight reads are shared-memory broadcasts); the weights of one temporal tap at a time sit
// in shared memory as [ky*7+kx][ci][64].  Zero padding (after the mean subtraction) outside the padded frame and the
// window's planes.
constexpr int kStemThreads = 128, kStemPx = 4;
template <typename T>
__global__ void stem_kernel(const float4* __restrict__ xin, int n_img, int TT, int Hp, int Wp, const float* __restrict__ w,
                            const float* __restrict__ bias, T* __restrict__ out) {
  __shared__ __align__(16) float ws[49 * 3 * 64];
  const int Ho = Hp / 2, Wo = Wp / 2, Wq = Wo / kStemPx;
  const size_t nquads = (size_t)n_img * Ho * Wq;
  const size_t total = 2 * ((nquads + 31) / 32) * 32;  // items: warps alternate between the two channel halves
  for (size_t base = (size_t)blockIdx.x * blockDim.x; base < total; base += (size_t)gridDim.x * blockDim.x) {
    const size_t it = base + threadIdx.x;
    const size_t wq = it >> 5;
    const int h = (int)(wq & 1);
    const size_t quad = (wq >> 1) * 32 + (it & 31);
    const bool valid = it < total && quad < nquads;
    const int img = valid ? (int)(quad / ((size_t)Ho * Wq)) : 0;
    const int rem = valid ? (int)(quad - (size_t)img * Ho * Wq) : 0;
    const int oy = rem / Wq, ox0 = (rem - oy * Wq) * kStemPx;
    const int t = img % TT;
    float acc[kStemPx][32];
#pragma unroll
    for (int c = 0; c < 32; ++c) {
      const float b0 = bias[h * 32 + c];
#pragma unroll
      for (int j = 0; j < kStemPx; ++j) acc[j][c] = b0;
    }
    for (int dt = 0; dt < 3; ++dt) {
      __syncthreads();
      for (int i = threadIdx.x; i < 49 * 3 * 64; i += blockDim.x) {
        const int co = i & 63, r = i >> 6, ci = r % 3, tap = r / 3;  // w [co][ci][dt][ky][kx]
        ws[i] = w[((co * 3 + ci) * 3 + dt) * 49 + tap];
      }
      __syncthreads();
      const int pl = t + dt - 1;
      if (!valid || pl < 0 || pl >= TT) continue;
      const float4* src = xin + (size_t)(img + dt - 1) * Hp * Wp;
      for (int ky = 0; ky < 7; ++ky) {
        const int y = 2 * oy + ky - 3;
        if (y < 0 || y >= Hp) continue;
        for (int kx = 0; kx < 7; ++kx) {
          float4 v[kStemPx];
#pragma unroll
          for (int j = 0; j < kStemPx; ++j) {
            const int x = 2 * (ox0 + j) + kx - 3;
            v[j] = (x >= 0 && x < Wp) ? src[(size_t)y * Wp + x] : make_float4(0.f, 0.f, 0.f, 0.f);
          }
          const float4* wt = reinterpret_cast<const float4*>(ws + (ky * 7 + kx) * 192 + h * 32);
#pragma unroll
          for (int c4 = 0; c4 < 8; ++c4) {
            const float4 w0 = wt[c4], w1 = wt[16 + c4], w2 = wt[32 + c4];  // ci = 0, 1, 2
            const float a0[4] = {w0.x, w0.y, w0.z, w0.w}, a1[4] = {w1.x, w1.y, w1.z, w1.w}, a2[4] = {w2.x, w2.y, w2.z, w2.w};
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
              for (int j = 0; j < kStemPx; ++j)
                acc[j][4 * c4 + e] = fmaf(v[j].z, a2[e], fmaf(v[j].y, a1[e], fmaf(v[j].x, a0[e], acc[j][4 * c4 + e])));
          }
        }
      }
    }
    if (!valid) continue;
#pragma unroll
    for (int j = 0; j < kStemPx; ++j) {
      T* o = out + ((size_t)img * Ho * Wo + (size_t)oy * Wo + ox0 + j) * 64 + h * 32;
#pragma unroll
      for (int c = 0; c < 32; c += 8) {
        float f[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = fmaxf(acc[j][c + e], 0.f);
        st8<T>(o + c, f);
      }
    }
  }
}

// partial[s][chunk][c] = sum over the chunk's pixels of sample s (npx pixels per sample) of x[.., c]; one thread per
// (s, chunk, 8 channels)
template <typename T>
__global__ void chan_sums_kernel(const T* __restrict__ x, int C, size_t npx, int S, int nchunk, float* __restrict__ partial) {
  const int nq = C / 8;
  const size_t total = (size_t)S * nchunk * nq;
  const size_t len = (npx + nchunk - 1) / nchunk;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = (int)(i % nq);
    const size_t sc = i / nq;
    const int chunk = (int)(sc % nchunk), s = (int)(sc / nchunk);
    const size_t p0 = (size_t)chunk * len, p1 = p0 + len < npx ? p0 + len : npx;
    float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const T* base = x + ((size_t)s * npx) * C + q * 8;
    for (size_t p = p0; p < p1; ++p) {
      float f[8];
      ld8<T>(base + p * C, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] += f[j];
    }
    float* d = partial + sc * C + q * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] = a[j];
  }
}

// g[s][c] = sigmoid(b[c] + sum_j W[c][j] mean[s][j]); mean[s][j] = sum over chunks and the `groups` channel groups of the
// partial sums (the four phases of a transposed conv) / count.  One block per sample (grid-stride).
__global__ void gate_kernel(const float* __restrict__ partial, int nchunk, int groups, int C, float inv_count,
                            const float* __restrict__ w, const float* __restrict__ b, int S, float* __restrict__ g) {
  __shared__ float mean[512];
  const int Ct = C * groups;
  for (int s = blockIdx.x; s < S; s += gridDim.x) {
    for (int j = threadIdx.x; j < C; j += blockDim.x) {
      float a = 0.f;
      for (int k = 0; k < nchunk; ++k)
        for (int q = 0; q < groups; ++q) a += partial[((size_t)s * nchunk + k) * Ct + q * C + j];
      mean[j] = a * inv_count;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      float a = b[c];
      for (int j = 0; j < C; ++j) a = fmaf(w[(size_t)c * C + j], mean[j], a);
      g[(size_t)s * C + c] = 1.f / (1.f + expf(-a));
    }
    __syncthreads();
  }
}

// out[img, y, x, c] = act(x[..] * g[img / T][c] (+ res[img, y, x, c])); phases: x holds the four phase outputs of a
// transposed conv at half resolution, [img][H/2][W/2][4 C] with phase (y & 1) * 2 + (x & 1); s2d (optional) also gets the
// result as [img][H/2][W/2][4 C], phase (y & 1) * 2 + (x & 1).  act 1 = ReLU, 2 = LeakyReLU(0.2).
template <typename T>
__global__ void apply_kernel(const T* __restrict__ x, int phases, const float* __restrict__ g, const T* __restrict__ res,
                             int act, T* __restrict__ out, T* __restrict__ s2d, int C, int n_img, int TT, int H, int W) {
  const int nq = C / 8;
  const size_t total = (size_t)n_img * H * W * nq;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = (int)(i % nq);
    const size_t pix = i / nq;
    const int xx = (int)(pix % W);
    const size_t r = pix / W;
    const int yy = (int)(r % H), img = (int)(r / H);
    const int ph = (yy & 1) * 2 + (xx & 1);
    const size_t half = (((size_t)img * (H / 2) + (yy >> 1)) * (W / 2) + (xx >> 1)) * (4 * C) + ph * C + q * 8;
    const T* src = phases ? x + half : x + pix * C + q * 8;
    float f[8];
    ld8<T>(src, f);
    const float* gg = g + (size_t)(img / TT) * C + q * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] *= gg[j];
    if (res) {
      float rr[8];
      ld8<T>(res + pix * C + q * 8, rr);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] += rr[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = act == 1 ? fmaxf(f[j], 0.f) : (f[j] > 0.f ? f[j] : 0.2f * f[j]);
    st8<T>(out + pix * C + q * 8, f);
    if (s2d) st8<T>(s2d + half, f);
  }
}

// outconv: one thread per output pixel of the unpadded frame; weights of the first 3 output channels in shared memory
// as [ky*7+kx][ci][3]
template <typename T>
__global__ void outconv_kernel(const T* __restrict__ x, int S, int Hp, int Wp, int H, int W, int pt, int pl,
                               const float* __restrict__ w, const float* __restrict__ bias, const float* __restrict__ sums,
                               int TT, float inv_count, float* __restrict__ out) {
  __shared__ float ws[49 * 64 * 3];
  for (int i = threadIdx.x; i < 49 * 64 * 3; i += blockDim.x) {
    const int co = i % 3, r = i / 3, ci = r & 63, tap = r >> 6;
    ws[i] = w[(co * 64 + ci) * 49 + tap];
  }
  __syncthreads();
  const size_t total = (size_t)S * H * W;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int xo = (int)(i % W);
    const size_t r = i / W;
    const int yo = (int)(r % H), s = (int)(r / H);
    float a[3] = {bias[0], bias[1], bias[2]};
    const T* base = x + (size_t)s * Hp * Wp * 64;
    for (int ky = 0; ky < 7; ++ky) {
      int y = yo + pt + ky - 3;
      y = y < 0 ? -y : (y >= Hp ? 2 * Hp - 2 - y : y);
      for (int kx = 0; kx < 7; ++kx) {
        int xx = xo + pl + kx - 3;
        xx = xx < 0 ? -xx : (xx >= Wp ? 2 * Wp - 2 - xx : xx);
        const T* p = base + ((size_t)y * Wp + xx) * 64;
        const float* wt = ws + (ky * 7 + kx) * 192;
#pragma unroll
        for (int c = 0; c < 64; c += 8) {
          float f[8];
          ld8<T>(p + c, f);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            a[0] = fmaf(f[j], wt[(c + j) * 3], a[0]);
            a[1] = fmaf(f[j], wt[(c + j) * 3 + 1], a[1]);
            a[2] = fmaf(f[j], wt[(c + j) * 3 + 2], a[2]);
          }
        }
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) out[i * 3 + c] = a[c] + window_mean(sums, s, c, TT, inv_count);
  }
}

}  // namespace

cudaError_t launch_flavr_frame_sums(const float* frames, int cstride, const FlavrFrameIdx& idx, int n_img, int H, int W,
                                    int Hp, int Wp, int pt, int pl, float* sums, cudaStream_t st) {
  VFI_LAUNCH(frame_sums_kernel, n_img, 256, 0, st, frames, cstride, idx, n_img, H, W, Hp, Wp, pt, pl, sums);
  return cudaGetLastError();
}

cudaError_t launch_flavr_prep(const float* frames, int cstride, const FlavrFrameIdx& idx, int n_img, int T, int H, int W,
                              int Hp, int Wp, int pt, int pl, const float* sums, float4* out, cudaStream_t st) {
  const float inv = 1.f / ((float)T * Hp * Wp);
  VFI_LAUNCH(prep_kernel, fl_grid((size_t)n_img * Hp * Wp, 256), 256, 0, st, frames, cstride, idx, n_img, T, H, W, Hp, Wp, pt,
             pl, sums, inv, out);
  return cudaGetLastError();
}

cudaError_t launch_flavr_stem(int op_type, const float4* xin, int n_img, int T, int Hp, int Wp, const float* w,
                              const float* bias, void* out, cudaStream_t st) {
  if ((Wp / 2) % kStemPx) return cudaErrorInvalidValue;
  const size_t quads = (size_t)n_img * (Hp / 2) * (Wp / 2 / kStemPx);
  const int g = fl_grid(2 * ((quads + 31) / 32) * 32, kStemThreads);
  if (op_type == OP_BF16)
    VFI_LAUNCH(stem_kernel<__nv_bfloat16>, g, kStemThreads, 0, st, xin, n_img, T, Hp, Wp, w, bias, (__nv_bfloat16*)out);
  else
    VFI_LAUNCH(stem_kernel<__half>, g, kStemThreads, 0, st, xin, n_img, T, Hp, Wp, w, bias, (__half*)out);
  return cudaGetLastError();
}

int flavr_sum_chunks(size_t npx) {
  const size_t c = (npx + 511) / 512;
  return (int)(c < 1 ? 1 : (c > 1024 ? 1024 : c));
}

cudaError_t launch_flavr_chan_sums(int op_type, const void* x, int C, size_t npx, int S, float* partial, cudaStream_t st) {
  if (C & 7) return cudaErrorInvalidValue;
  const int nchunk = flavr_sum_chunks(npx);
  const int g = fl_grid((size_t)S * nchunk * (C / 8), 128);
  if (op_type == OP_BF16)
    VFI_LAUNCH(chan_sums_kernel<__nv_bfloat16>, g, 128, 0, st, (const __nv_bfloat16*)x, C, npx, S, nchunk, partial);
  else
    VFI_LAUNCH(chan_sums_kernel<__half>, g, 128, 0, st, (const __half*)x, C, npx, S, nchunk, partial);
  return cudaGetLastError();
}

cudaError_t launch_flavr_gate(const float* partial, size_t npx, int groups, int C, size_t count, const float* w,
                              const float* b, int S, float* g, cudaStream_t st) {
  if (C > 512) return cudaErrorInvalidValue;
  VFI_LAUNCH(gate_kernel, S, 256, 0, st, partial, flavr_sum_chunks(npx), groups, C, (float)(1.0 / (double)count), w, b, S, g);
  return cudaGetLastError();
}

cudaError_t launch_flavr_apply(int op_type, const void* x, int phases, const float* g, const void* res, int act, void* out,
                               void* s2d, int C, int n_img, int T, int H, int W, cudaStream_t st) {
  if ((C & 7) || ((phases || s2d) && ((H | W) & 1))) return cudaErrorInvalidValue;
  const int gr = fl_grid((size_t)n_img * H * W * (C / 8), 256);
  if (op_type == OP_BF16)
    VFI_LAUNCH(apply_kernel<__nv_bfloat16>, gr, 256, 0, st, (const __nv_bfloat16*)x, phases, g, (const __nv_bfloat16*)res, act,
               (__nv_bfloat16*)out, (__nv_bfloat16*)s2d, C, n_img, T, H, W);
  else
    VFI_LAUNCH(apply_kernel<__half>, gr, 256, 0, st, (const __half*)x, phases, g, (const __half*)res, act, (__half*)out,
               (__half*)s2d, C, n_img, T, H, W);
  return cudaGetLastError();
}

cudaError_t launch_flavr_outconv(int op_type, const void* x, int S, int Hp, int Wp, int H, int W, int pt, int pl,
                                 const float* w, const float* bias, const float* sums, int T, float* out, cudaStream_t st) {
  const float inv = 1.f / ((float)T * Hp * Wp);
  const int g = fl_grid((size_t)S * H * W, 128);
  if (op_type == OP_BF16)
    VFI_LAUNCH(outconv_kernel<__nv_bfloat16>, g, 128, 0, st, (const __nv_bfloat16*)x, S, Hp, Wp, H, W, pt, pl, w, bias, sums, T,
               inv, out);
  else
    VFI_LAUNCH(outconv_kernel<__half>, g, 128, 0, st, (const __half*)x, S, Hp, Wp, H, W, pt, pl, w, bias, sums, T, inv, out);
  return cudaGetLastError();
}

}  // namespace vfi
