// The kernels of the CAIN path (cain.cu) around its tensor-core convolutions, on the CUDA cores.
// Activations are 16-bit NHWC tensors on the bordered grid: the h x w grid of the 1/8-resolution trunk stored on
// (h + 2) x (w + 2) cells, grid cell (y, x) at cell (y + 1, x + 1), 192 channels per cell (the prep output: 384, frame 0's
// channels then frame 1's).  The frames and the output are fp32 [3][H][W] planes.  Reference: vfi_models/cain/
// cain_arch.py, common.py.
//
//   frame_sums   per-(frame, channel) partial sums over the unpadded frames, in double   sub_mean
//   prep         (frame - mean), reflection padding to hp x wp, space-to-depth by 8,    InOutPaddings, pixel_shuffle(1/8)
//                zero border (headConv pads with zeros)
//   border       the border cells as ReflectionPad2d(1) of the interior (ConvNorm), or zero with an optional sum
//                added to the interior (res = body(x) + x before tailConv)
//   chan_sums    per-(interior row, channel) sums of a conv output                      CALayer.avg_pool
//   gate         sigmoid(W2 relu(W1 mean + b1) + b2) in fp32                           CALayer.conv_du
//   apply        x * gate + residual on every cell, the border from the reflected cell   RCAB: out = body(x) + x
//   final        depth-to-space by 8, crop, + (m0 + m1) / 2                              pixel_shuffle(8), paddingOutput
#include "ptx.cuh"
#include "vfi_internal.h"

namespace vfi {

namespace {

constexpr int kQ = kCainChannels / 8;  // 8-channel vectors per cell

inline int cain_grid(size_t total, int threads) {
  size_t b = (total + threads - 1) / threads;
  return (int)(b < 1 ? 1 : (b > 1048576 ? 1048576 : b));
}

template <typename T>
__device__ __forceinline__ void cain_ld8(const T* p, float (&f)[8]) {
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
__device__ __forceinline__ void cain_st8(T* p, const float (&f)[8]) {
  uint4 u;
  u.x = Pack2<T>::pack(f[0], f[1]);
  u.y = Pack2<T>::pack(f[2], f[3]);
  u.z = Pack2<T>::pack(f[4], f[5]);
  u.w = Pack2<T>::pack(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// ReflectionPad2d index: -i before the axis, 2 (n - 1) - i after it (the padding is smaller than n)
__device__ __forceinline__ int cain_reflect(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * (n - 1) - i : i); }

// the cell a border cell of a (h + 2) x (w + 2) grid mirrors under ReflectionPad2d(1): row 0 -> 2, row h + 1 -> h - 1
__device__ __forceinline__ int cain_mirror(int i, int n) { return i == 0 ? 2 : (i == n + 1 ? n - 1 : i); }

// ---------------------------------------------------------------- means
// partial[plane * kCainMeanChunks + k]: chunk k of plane (frame * 3 + channel); one block per item (grid-stride)
__global__ void cain_frame_sums_kernel(const float* __restrict__ f0, const float* __restrict__ f1, int npx,
                                       double* __restrict__ partial) {
  __shared__ double red[256];
  const int len = (npx + kCainMeanChunks - 1) / kCainMeanChunks;
  for (int item = blockIdx.x; item < 6 * kCainMeanChunks; item += gridDim.x) {
    const int plane = item / kCainMeanChunks, k = item - plane * kCainMeanChunks;
    const float* src = (plane < 3 ? f0 : f1) + (size_t)(plane % 3) * npx;
    const int p0 = k * len, p1 = p0 + len < npx ? p0 + len : npx;
    double a = 0.0;
    for (int p = p0 + threadIdx.x; p < p1; p += blockDim.x) a += (double)src[p];
    red[threadIdx.x] = a;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
      if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
      __syncthreads();
    }
    if (threadIdx.x == 0) partial[item] = red[0];
    __syncthreads();
  }
}

// m[frame * 3 + c]: the six means, reduced in a fixed order by every block that needs them
__device__ __forceinline__ void cain_means(const double* __restrict__ partial, int npx, float* m) {
  for (int j = threadIdx.x; j < 6; j += blockDim.x) {
    double s = 0.0;
    for (int k = 0; k < kCainMeanChunks; ++k) s += partial[j * kCainMeanChunks + k];
    m[j] = (float)(s / (double)npx);
  }
  __syncthreads();
}

// ---------------------------------------------------------------- prep
// one item = (cell, frame, channel, sub-pixel row sy): 8 sub-pixel columns, 16 bytes of the 384-channel output
template <typename T>
__global__ void cain_prep_kernel(const float* __restrict__ f0, const float* __restrict__ f1, int H, int W, int top,
                                 int left, int h, int w, const double* __restrict__ partial, T* __restrict__ out) {
  __shared__ float m[6];
  cain_means(partial, H * W, m);
  const int wb = w + 2;
  const size_t total = (size_t)(h + 2) * wb * 48;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int sy = (int)(i & 7), fc = (int)((i >> 3) % 6);
    const size_t cell = (i >> 3) / 6;
    const int yy = (int)(cell / wb), xx = (int)(cell - (size_t)yy * wb);
    const int f = fc / 3, c = fc - 3 * f;
    float v[8];
    if (yy == 0 || xx == 0 || yy == h + 1 || xx == w + 1) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = 0.f;
    } else {
      const int y = cain_reflect((yy - 1) * 8 + sy - top, H);
      const float* row = (f ? f1 : f0) + ((size_t)c * H + y) * W;
      const float mu = m[fc];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = row[cain_reflect((xx - 1) * 8 + j - left, W)] - mu;
    }
    cain_st8<T>(out + cell * (2 * kCainChannels) + f * kCainChannels + c * 64 + sy * 8, v);
  }
}

// ---------------------------------------------------------------- border
// reflect: each border cell (8 channels per item) copies the cell it mirrors
template <typename T>
__global__ void cain_border_reflect_kernel(T* __restrict__ x, int h, int w) {
  const int wb = w + 2, nb = 2 * wb + 2 * h;
  const size_t total = (size_t)nb * kQ;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = (int)(i % kQ), b = (int)(i / kQ);
    int yy, xx;
    if (b < wb) {
      yy = 0, xx = b;
    } else if (b < 2 * wb) {
      yy = h + 1, xx = b - wb;
    } else {
      const int r = b - 2 * wb;
      yy = 1 + (r >> 1), xx = (r & 1) ? w + 1 : 0;
    }
    const int sy = cain_mirror(yy, h), sx = cain_mirror(xx, w);
    const uint4 v = *reinterpret_cast<const uint4*>(x + ((size_t)sy * wb + sx) * kCainChannels + q * 8);
    *reinterpret_cast<uint4*>(x + ((size_t)yy * wb + xx) * kCainChannels + q * 8) = v;
  }
}

// zero: the border cells become 0; with `add`, every interior cell gets x + add (in place, one owner per element)
template <typename T>
__global__ void cain_border_zero_kernel(T* __restrict__ x, const T* __restrict__ add, int h, int w) {
  const int wb = w + 2;
  const size_t total = (size_t)(h + 2) * wb * kQ;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t cell = i / kQ;
    const int yy = (int)(cell / wb), xx = (int)(cell - (size_t)yy * wb);
    T* p = x + i * 8;
    if (yy == 0 || xx == 0 || yy == h + 1 || xx == w + 1) {
      *reinterpret_cast<uint4*>(p) = make_uint4(0u, 0u, 0u, 0u);
    } else if (add) {
      float a[8], b[8];
      cain_ld8<T>(p, a);
      cain_ld8<T>(add + i * 8, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] += b[j];
      cain_st8<T>(p, a);
    }
  }
}

// ---------------------------------------------------------------- channel attention
// partial[row][c] = sum over the interior cells of grid row `row` of x[.., c]; a block per row (grid-stride), its
// threads as 8 cell lanes x 24 channel vectors, the lanes summed in a fixed order
template <typename T>
__global__ void cain_chan_sums_kernel(const T* __restrict__ x, int h, int w, float* __restrict__ partial) {
  __shared__ float red[8][kCainChannels];
  const int wb = w + 2;
  for (int row = blockIdx.x; row < h; row += gridDim.x) {
    for (int v = threadIdx.x; v < 8 * kQ; v += blockDim.x) {
      const int lane = v / kQ, q = v - lane * kQ;
      float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      const T* base = x + ((size_t)(row + 1) * wb + 1) * kCainChannels + q * 8;
      for (int gx = lane; gx < w; gx += 8) {
        float f[8];
        cain_ld8<T>(base + (size_t)gx * kCainChannels, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] += f[j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) red[lane][q * 8 + j] = a[j];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < kCainChannels; c += blockDim.x) {
      float s = 0.f;
      for (int lane = 0; lane < 8; ++lane) s += red[lane][c];
      partial[(size_t)row * kCainChannels + c] = s;
    }
    __syncthreads();
  }
}

// g[c] = sigmoid(b2[c] + sum_j W2[c][j] relu(b1[j] + sum_k W1[j][k] mean[k])); ca = {W1 [12][192], b1 [12],
// W2 [192][12], b2 [192]}.  One block.
__global__ void cain_gate_kernel(const float* __restrict__ partial, int h, float inv_count, const float* __restrict__ ca,
                                 float* __restrict__ g) {
  __shared__ float mean[kCainChannels];
  __shared__ float hid[kCainHidden];
  const float* w1 = ca;
  const float* b1 = w1 + kCainHidden * kCainChannels;
  const float* w2 = b1 + kCainHidden;
  const float* b2 = w2 + kCainChannels * kCainHidden;
  for (int c = threadIdx.x; c < kCainChannels; c += blockDim.x) {
    float s = 0.f;
    for (int r = 0; r < h; ++r) s += partial[(size_t)r * kCainChannels + c];
    mean[c] = s * inv_count;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < kCainHidden; j += blockDim.x) {
    float a = b1[j];
    for (int k = 0; k < kCainChannels; ++k) a = fmaf(w1[j * kCainChannels + k], mean[k], a);
    hid[j] = fmaxf(a, 0.f);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < kCainChannels; c += blockDim.x) {
    float a = b2[c];
    for (int j = 0; j < kCainHidden; ++j) a = fmaf(w2[c * kCainHidden + j], hid[j], a);
    g[c] = 1.f / (1.f + expf(-a));
  }
}

// out[cell] = x[m] * g + res[m], m = the cell itself inside, the mirrored interior cell on the border: the result's
// border is ReflectionPad2d(1) of its interior, ready for the next ConvNorm
template <typename T>
__global__ void cain_apply_kernel(const T* __restrict__ x, const float* __restrict__ g, const T* __restrict__ res,
                                  T* __restrict__ out, int h, int w) {
  const int wb = w + 2;
  const size_t total = (size_t)(h + 2) * wb * kQ;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = (int)(i % kQ);
    const size_t cell = i / kQ;
    const int yy = (int)(cell / wb), xx = (int)(cell - (size_t)yy * wb);
    const size_t src = ((size_t)cain_mirror(yy, h) * wb + cain_mirror(xx, w)) * kCainChannels + q * 8;
    float a[8], r[8];
    cain_ld8<T>(x + src, a);
    cain_ld8<T>(res + src, r);
    const float* gg = g + q * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = fmaf(a[j], gg[j], r[j]);
    cain_st8<T>(out + i * 8, a);
  }
}

// ---------------------------------------------------------------- final
template <typename T>
__global__ void cain_final_kernel(const T* __restrict__ feat, int H, int W, int top, int left, int w,
                                  const double* __restrict__ partial, float* __restrict__ out) {
  __shared__ float m[6];
  cain_means(partial, H * W, m);
  const int wb = w + 2;
  const size_t total = (size_t)3 * H * W;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const size_t r = i / W;
    const int y = (int)(r % H), c = (int)(r / H);
    const int py = y + top, px = x + left;
    const size_t cell = (size_t)((py >> 3) + 1) * wb + (px >> 3) + 1;
    const float v = (float)feat[cell * kCainChannels + c * 64 + (py & 7) * 8 + (px & 7)];
    out[i] = v + (m[c] + m[3 + c]) / 2.f;
  }
}

}  // namespace

cudaError_t launch_cain_frame_sums(const float* f0, const float* f1, int H, int W, double* partial, cudaStream_t st) {
  VFI_LAUNCH(cain_frame_sums_kernel, 6 * kCainMeanChunks, 256, 0, st, f0, f1, H * W, partial);
  return cudaGetLastError();
}

cudaError_t launch_cain_prep(int op, const float* f0, const float* f1, int H, int W, int top, int left, int h, int w,
                             const double* partial, void* out, cudaStream_t st) {
  const int g = cain_grid((size_t)(h + 2) * (w + 2) * 48, 256);
  if (op == OP_BF16)
    VFI_LAUNCH(cain_prep_kernel<__nv_bfloat16>, g, 256, 0, st, f0, f1, H, W, top, left, h, w, partial, (__nv_bfloat16*)out);
  else
    VFI_LAUNCH(cain_prep_kernel<__half>, g, 256, 0, st, f0, f1, H, W, top, left, h, w, partial, (__half*)out);
  return cudaGetLastError();
}

cudaError_t launch_cain_border(int op, void* x, const void* add, int h, int w, bool reflect, cudaStream_t st) {
  if (reflect && add) return cudaErrorInvalidValue;
  if (reflect) {
    const int g = cain_grid((size_t)(2 * (w + 2) + 2 * h) * kQ, 256);
    if (op == OP_BF16)
      VFI_LAUNCH(cain_border_reflect_kernel<__nv_bfloat16>, g, 256, 0, st, (__nv_bfloat16*)x, h, w);
    else
      VFI_LAUNCH(cain_border_reflect_kernel<__half>, g, 256, 0, st, (__half*)x, h, w);
  } else {
    const int g = cain_grid((size_t)(h + 2) * (w + 2) * kQ, 256);
    if (op == OP_BF16)
      VFI_LAUNCH(cain_border_zero_kernel<__nv_bfloat16>, g, 256, 0, st, (__nv_bfloat16*)x, (const __nv_bfloat16*)add, h, w);
    else
      VFI_LAUNCH(cain_border_zero_kernel<__half>, g, 256, 0, st, (__half*)x, (const __half*)add, h, w);
  }
  return cudaGetLastError();
}

cudaError_t launch_cain_chan_sums(int op, const void* x, int h, int w, float* partial, cudaStream_t st) {
  if (op == OP_BF16)
    VFI_LAUNCH(cain_chan_sums_kernel<__nv_bfloat16>, h, 8 * kQ, 0, st, (const __nv_bfloat16*)x, h, w, partial);
  else
    VFI_LAUNCH(cain_chan_sums_kernel<__half>, h, 8 * kQ, 0, st, (const __half*)x, h, w, partial);
  return cudaGetLastError();
}

cudaError_t launch_cain_gate(const float* partial, int h, int w, const float* ca, float* g, cudaStream_t st) {
  VFI_LAUNCH(cain_gate_kernel, 1, kCainChannels, 0, st, partial, h, (float)(1.0 / ((double)h * w)), ca, g);
  return cudaGetLastError();
}

cudaError_t launch_cain_apply(int op, const void* x, const float* g, const void* res, void* out, int h, int w,
                              cudaStream_t st) {
  const int gr = cain_grid((size_t)(h + 2) * (w + 2) * kQ, 256);
  if (op == OP_BF16)
    VFI_LAUNCH(cain_apply_kernel<__nv_bfloat16>, gr, 256, 0, st, (const __nv_bfloat16*)x, g, (const __nv_bfloat16*)res,
               (__nv_bfloat16*)out, h, w);
  else
    VFI_LAUNCH(cain_apply_kernel<__half>, gr, 256, 0, st, (const __half*)x, g, (const __half*)res, (__half*)out, h, w);
  return cudaGetLastError();
}

cudaError_t launch_cain_final(int op, const void* feat, int H, int W, int top, int left, int w, const double* partial,
                              float* out, cudaStream_t st) {
  const int g = cain_grid((size_t)3 * H * W, 256);
  if (op == OP_BF16)
    VFI_LAUNCH(cain_final_kernel<__nv_bfloat16>, g, 256, 0, st, (const __nv_bfloat16*)feat, H, W, top, left, w, partial, out);
  else
    VFI_LAUNCH(cain_final_kernel<__half>, g, 256, 0, st, (const __half*)feat, H, W, top, left, w, partial, out);
  return cudaGetLastError();
}

}  // namespace vfi
