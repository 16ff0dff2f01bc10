// The kernels of the IFRNet path (ifrnet.cu) around its tensor-core convolutions, on the CUDA cores.
// Activations are 16-bit NHWC tensors (image 0 = frame 0, image 1 = frame 1 in the encoder; one image in the decoders);
// flows, mask, warps and the blend are fp32.  Reference: vfi_models/ifrnet/IFRNet_{S,L}_arch.py.
//
//   frame_sums   partial sums of both frames (the zero padding adds nothing)          mean_ (IRFNet.forward)
//   prep         (padded frame - mean_) resized by the resize factor, as float4 planes  resize(img0 - mean_, t)
//   first_conv   encoder.pyramid1.0: Conv2d(3, c, 3 / 7, stride 2, pad 1 / 3) + PReLU
//   s2d          the space-to-depth copy a stride-2 conv (pyramid2..4.0) reads as a 2x2 conv
//   dec4_in      cat(f0_4, f1_4, embt plane) in the padded channel layout of decoder 4
//   dec_flow     interleave the fp32 phases of a decoder's ConvT, + 2 * resize(previous flow, 2) (sigmoid on the mask)
//   dec_in       cat(ft_, warp(f0, flow0), warp(f1, flow1), flow0, flow1) in the padded layout of decoders 3..1
//   final        resize(flow, mask, res; 1/t), two fp32 image warps, merge, + mean_ + res, clamp, crop
#include "ptx.cuh"
#include "vfi_internal.h"

namespace vfi {

namespace {

inline int ifr_grid(size_t total, int threads) {
  size_t b = (total + threads - 1) / threads;
  return (int)(b < 1 ? 1 : (b > 1048576 ? 1048576 : b));
}

template <typename T>
__device__ __forceinline__ void ifr_ld8(const T* p, float (&f)[8]) {
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
__device__ __forceinline__ void ifr_st8(T* p, const float (&f)[8]) {
  uint4 u;
  u.x = Pack2<T>::pack(f[0], f[1]);
  u.y = Pack2<T>::pack(f[2], f[3]);
  u.z = Pack2<T>::pack(f[4], f[5]);
  u.w = Pack2<T>::pack(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// F.interpolate(bilinear, align_corners=False) source index along one axis: src = scale * (dst + 0.5) - 0.5 with the
// scale 1 / scale_factor (fp32), clamped at 0; i1 = i0 + 1 unless i0 is the last row
struct Lin {
  int i0, i1;
  float l0, l1;
};
__device__ __forceinline__ Lin ifr_lin(float scale, int dst, int in_size) {
  float src = scale * ((float)dst + 0.5f) - 0.5f;
  if (src < 0.f) src = 0.f;
  Lin r;
  r.i0 = (int)src;
  if (r.i0 > in_size - 1) r.i0 = in_size - 1;
  r.i1 = r.i0 + (r.i0 < in_size - 1 ? 1 : 0);
  r.l1 = src - (float)r.i0;
  if (r.l1 > 1.f) r.l1 = 1.f;
  r.l0 = 1.f - r.l1;
  return r;
}

// torch.linspace(-1, 1, n)[i] in fp32
__device__ __forceinline__ float ifr_linspace(int i, int n) {
  const float step = 2.0f / (float)(n - 1);
  return i < n / 2 ? -1.f + step * (float)i : 1.f - step * (float)(n - 1 - i);
}

// warp(): the grid comes from the flow's size (gw x gh), grid_sample(bilinear, border, align_corners=True) reads an image
// of its own size (iw x ih).  Returns the four corner indices (-1: outside, weight skipped) and weights.
struct Tap4 {
  int x0, y0, x1, y1;
  float w00, w01, w10, w11;
};
__device__ __forceinline__ Tap4 ifr_warp_taps(int X, int Y, int gw, int gh, float fx, float fy, int iw, int ih) {
  const float gx = ifr_linspace(X, gw) + fx / (((float)gw - 1.0f) / 2.0f);
  const float gy = ifr_linspace(Y, gh) + fy / (((float)gh - 1.0f) / 2.0f);
  float ix = ((gx + 1.f) / 2.f) * (float)(iw - 1);
  float iy = ((gy + 1.f) / 2.f) * (float)(ih - 1);
  ix = fminf(fmaxf(ix, 0.f), (float)(iw - 1));
  iy = fminf(fmaxf(iy, 0.f), (float)(ih - 1));
  Tap4 t;
  const float fx0 = floorf(ix), fy0 = floorf(iy);
  t.x0 = (int)fx0;
  t.y0 = (int)fy0;
  const float ax = ix - fx0, ay = iy - fy0;
  t.w00 = (1.f - ax) * (1.f - ay);
  t.w01 = ax * (1.f - ay);
  t.w10 = (1.f - ax) * ay;
  t.w11 = ax * ay;
  t.x1 = t.x0 + 1 < iw ? t.x0 + 1 : -1;
  t.y1 = t.y0 + 1 < ih ? t.y0 + 1 : -1;
  return t;
}

// ---------------------------------------------------------------- mean_
__global__ void ifr_frame_sums_kernel(const float* __restrict__ f0, const float* __restrict__ f1, size_t n,
                                      double* __restrict__ partial) {
  double a = 0.0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    a += (double)f0[i] + (double)f1[i];
  __shared__ double red[256];
  red[threadIdx.x] = a;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.x] = red[0];
}

__global__ void ifr_mean_kernel(const double* __restrict__ partial, int nparts, double count, float* __restrict__ mean) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < nparts; ++i) s += partial[i];
    mean[0] = (float)(s / count);
  }
}

// ---------------------------------------------------------------- encoder input
// out[img][y][x] = bilinear resize of (padded frame img - mean_) to h0 x w0; the padding reads as 0 - mean_
__global__ void ifr_prep_kernel(const float* __restrict__ f0, const float* __restrict__ f1, int H, int W, int Hp, int Wp,
                                int h0, int w0, float scale, const float* __restrict__ mean, float4* __restrict__ out) {
  const size_t hw = (size_t)h0 * w0, total = 2 * hw;
  const float m = mean[0];
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int img = (int)(i / hw);
    const int p = (int)(i - (size_t)img * hw);
    const int oy = p / w0, ox = p - oy * w0;
    const float* f = img ? f1 : f0;
    const Lin ly = ifr_lin(scale, oy, Hp), lx = ifr_lin(scale, ox, Wp);
    float v[3];
    for (int c = 0; c < 3; ++c) {
      const float* pl = f + (size_t)c * H * W;
      auto at = [&](int y, int x) { return (y < H && x < W) ? pl[(size_t)y * W + x] - m : -m; };
      v[c] = ly.l0 * (lx.l0 * at(ly.i0, lx.i0) + lx.l1 * at(ly.i0, lx.i1)) +
             ly.l1 * (lx.l0 * at(ly.i1, lx.i0) + lx.l1 * at(ly.i1, lx.i1));
    }
    out[i] = make_float4(v[0], v[1], v[2], 0.f);
  }
}

// pyramid1.0: Conv2d(3, C, k, stride 2, pad k / 2) + PReLU; a thread computes 8 output channels of one pixel and also
// zeroes the padding channels [C, pitch) of its 8-channel chunk
template <typename T>
__global__ void ifr_first_conv_kernel(const float4* __restrict__ xin, int h0, int w0, int h1, int w1, int k,
                                      const float* __restrict__ w, const float* __restrict__ bias,
                                      const float* __restrict__ slopes, int C, int pitch, T* __restrict__ out) {
  const int chunks = pitch / 8;
  const size_t total = (size_t)2 * h1 * w1 * chunks;
  const int pad = k / 2;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % chunks);
    const size_t pix = i / chunks;
    const int ox = (int)(pix % w1);
    const int oy = (int)((pix / w1) % h1);
    const int img = (int)(pix / ((size_t)w1 * h1));
    float acc[8];
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    const int c0 = ch * 8;
    if (c0 < C) {
      for (int j = 0; j < 8; ++j) acc[j] = c0 + j < C ? bias[c0 + j] : 0.f;
      const float4* src = xin + (size_t)img * h0 * w0;
      for (int ky = 0; ky < k; ++ky) {
        const int y = 2 * oy + ky - pad;
        if (y < 0 || y >= h0) continue;
        for (int kx = 0; kx < k; ++kx) {
          const int x = 2 * ox + kx - pad;
          if (x < 0 || x >= w0) continue;
          const float4 v = src[(size_t)y * w0 + x];
          for (int j = 0; j < 8; ++j) {
            if (c0 + j >= C) break;
            const float* wr = w + (size_t)(c0 + j) * 3 * k * k + ky * k + kx;
            acc[j] = fmaf(v.x, wr[0], acc[j]);
            acc[j] = fmaf(v.y, wr[k * k], acc[j]);
            acc[j] = fmaf(v.z, wr[2 * k * k], acc[j]);
          }
        }
      }
      for (int j = 0; j < 8; ++j)
        if (c0 + j < C) acc[j] = acc[j] > 0.f ? acc[j] : slopes[c0 + j] * acc[j];
    }
    ifr_st8(out + pix * pitch + c0, acc);
  }
}

// space-to-depth: out[b][Y][X][q * cq + c] = in[b][2Y + py][2X + px][c], q = py * 2 + px, cq = C rounded up to 8; zero
// outside the input and in the padding channels [4 cq, opitch)
template <typename T>
__global__ void ifr_s2d_kernel(const T* __restrict__ in, int pitch, int cq, int B, int h, int w, T* __restrict__ out,
                               int opitch) {
  const int ho = (h + 1) / 2, wo = (w + 1) / 2, chunks = opitch / 8, qc = cq / 8;
  const size_t total = (size_t)B * ho * wo * chunks;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % chunks);
    const size_t pix = i / chunks;
    const int X = (int)(pix % wo);
    const int Y = (int)((pix / wo) % ho);
    const int b = (int)(pix / ((size_t)wo * ho));
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    const int q = ch / qc;
    if (q < 4) {
      const int y = 2 * Y + (q >> 1), x = 2 * X + (q & 1);
      if (y < h && x < w) v = *reinterpret_cast<const uint4*>(in + (((size_t)b * h + y) * w + x) * pitch + (ch - q * qc) * 8);
    }
    *reinterpret_cast<uint4*>(out + pix * opitch + ch * 8) = v;
  }
}

// decoder 4 input: [f0_4 | f1_4 | embt, zeros] with groups at 0, g1 and g2 (pitch g2 + 64)
template <typename T>
__global__ void ifr_dec4_in_kernel(const T* __restrict__ f, int fpitch, int g1, int h, int w, float embt,
                                   T* __restrict__ out) {
  const int pitch = 2 * g1 + 64, chunks = pitch / 8;
  const size_t total = (size_t)h * w * chunks;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c0 = (int)(i % chunks) * 8;
    const size_t pix = i / chunks;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (c0 < 2 * g1) {
      const int img = c0 >= g1, c = c0 - img * g1;
      if (c < fpitch) v = *reinterpret_cast<const uint4*>(f + ((size_t)img * h * w + pix) * fpitch + c);
    } else if (c0 == 2 * g1) {
      float e[8] = {embt, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      ifr_st8(out + pix * pitch + c0, e);
      continue;
    }
    *reinterpret_cast<uint4*>(out + pix * pitch + c0) = v;
  }
}

// acc[Y][X][0..nf) on the grid 2h x 2w: phase (Y & 1, X & 1) of the ConvT's fp32 columns (ph [h][w][4][nf]); columns
// 0..3 (two flows) + 2 * resize(prev, 2) when prev is given ([h][w][4]); nf = 8: column 4 through a sigmoid (the mask)
__global__ void ifr_dec_flow_kernel(const float* __restrict__ ph, int nf, const float* __restrict__ prev, int h, int w,
                                    float* __restrict__ acc) {
  const int H2 = 2 * h, W2 = 2 * w;
  const size_t total = (size_t)H2 * W2;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int Y = (int)(i / W2), X = (int)(i - (size_t)Y * W2);
    const float* s = ph + (((size_t)(Y >> 1) * w + (X >> 1)) * 4 + (Y & 1) * 2 + (X & 1)) * nf;
    float v[8];
    for (int c = 0; c < nf; ++c) v[c] = s[c];
    if (prev) {
      const Lin ly = ifr_lin(0.5f, Y, h), lx = ifr_lin(0.5f, X, w);
      for (int c = 0; c < 4; ++c) {
        auto at = [&](int y, int x) { return prev[((size_t)y * w + x) * 4 + c]; };
        const float u = ly.l0 * (lx.l0 * at(ly.i0, lx.i0) + lx.l1 * at(ly.i0, lx.i1)) +
                        ly.l1 * (lx.l0 * at(ly.i1, lx.i0) + lx.l1 * at(ly.i1, lx.i1));
        v[c] = v[c] + 2.0f * u;
      }
    }
    if (nf == 8) v[4] = 1.f / (1.f + expf(-v[4]));
    for (int c = 0; c < nf; ++c) acc[i * nf + c] = v[c];
  }
}

// decoders 3..1 input on the grid gh x gw: [ft_ | warp(f0, flow0) | warp(f1, flow1) | flow0, flow1, zeros] with groups at
// 0, g1, g2, g3 (pitch g3 + 64).  ft_ = columns 8.. of the previous ConvT's 16-bit phases (ph16 [gh/2][gw/2][4][pp]),
// the features f [2][fh][fw][fpitch] are sampled at their own size, the flows come from acc ([gh][gw][4]).
template <typename T>
__global__ void ifr_dec_in_kernel(const T* __restrict__ ph16, int pp, const T* __restrict__ f, int fpitch, int fh, int fw,
                                  const float* __restrict__ acc, int gh, int gw, int g1, int g2, int g3,
                                  T* __restrict__ out) {
  const int pitch = g3 + 64, chunks = pitch / 8;
  const size_t total = (size_t)gh * gw * chunks;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c0 = (int)(i % chunks) * 8;
    const size_t pix = i / chunks;
    const int Y = (int)(pix / gw), X = (int)(pix - (size_t)Y * gw);
    T* o = out + pix * pitch + c0;
    float v[8];
    for (int j = 0; j < 8; ++j) v[j] = 0.f;
    if (c0 < g1) {
      const int c = 8 + c0;
      if (c < pp)
        *reinterpret_cast<uint4*>(o) = *reinterpret_cast<const uint4*>(
            ph16 + (((size_t)(Y >> 1) * (gw >> 1) + (X >> 1)) * 4 + (Y & 1) * 2 + (X & 1)) * pp + c);
      else
        *reinterpret_cast<uint4*>(o) = make_uint4(0u, 0u, 0u, 0u);
      continue;
    }
    const float* a = acc + pix * 4;
    if (c0 < g3) {
      const int img = c0 >= g2, c = c0 - (img ? g2 : g1);
      if (c < fpitch) {
        const Tap4 t = ifr_warp_taps(X, Y, gw, gh, a[2 * img], a[2 * img + 1], fw, fh);
        const T* src = f + (size_t)img * fh * fw * fpitch + c;
        float q[8];
        auto add = [&](int y, int x, float wt) {
          if (y < 0 || x < 0) return;
          ifr_ld8(src + ((size_t)y * fw + x) * fpitch, q);
          for (int j = 0; j < 8; ++j) v[j] += wt * q[j];
        };
        add(t.y0, t.x0, t.w00);
        add(t.y0, t.x1, t.w01);
        add(t.y1, t.x0, t.w10);
        add(t.y1, t.x1, t.w11);
      }
    } else if (c0 == g3) {
      for (int j = 0; j < 4; ++j) v[j] = a[j];
    }
    ifr_st8(o, v);
  }
}

// the frame: acc1 [hq][wq][8] (flow0, flow1, sigmoid(mask), res) resized by 1/t to hF x wF (only the H x W crop is
// computed), flows times 1/t, warps of the padded full-resolution frames minus mean_ (Hp x Wp), merge, clamp
__global__ void ifr_final_kernel(const float* __restrict__ f0, const float* __restrict__ f1, int H, int W, int Hp, int Wp,
                                 const float* __restrict__ acc, int hq, int wq, int hF, int wF, float scale, float fmul,
                                 const float* __restrict__ mean, float* __restrict__ out) {
  const size_t total = (size_t)H * W;
  const float m = mean[0];
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
    const Lin ly = ifr_lin(scale, y, hq), lx = ifr_lin(scale, x, wq);
    float r[8];
    for (int c = 0; c < 8; ++c) {
      auto at = [&](int yy, int xx) { return acc[((size_t)yy * wq + xx) * 8 + c]; };
      r[c] = ly.l0 * (lx.l0 * at(ly.i0, lx.i0) + lx.l1 * at(ly.i0, lx.i1)) +
             ly.l1 * (lx.l0 * at(ly.i1, lx.i0) + lx.l1 * at(ly.i1, lx.i1));
    }
    float wv[2][3];
    for (int k = 0; k < 2; ++k) {
      const float* img = k ? f1 : f0;
      const Tap4 t = ifr_warp_taps(x, y, wF, hF, r[2 * k] * fmul, r[2 * k + 1] * fmul, Wp, Hp);
      for (int c = 0; c < 3; ++c) {
        const float* pl = img + (size_t)c * H * W;
        auto at = [&](int yy, int xx) { return (yy < H && xx < W) ? pl[(size_t)yy * W + xx] - m : -m; };
        float s = 0.f;
        if (t.y0 >= 0 && t.x0 >= 0) s += t.w00 * at(t.y0, t.x0);
        if (t.y0 >= 0 && t.x1 >= 0) s += t.w01 * at(t.y0, t.x1);
        if (t.y1 >= 0 && t.x0 >= 0) s += t.w10 * at(t.y1, t.x0);
        if (t.y1 >= 0 && t.x1 >= 0) s += t.w11 * at(t.y1, t.x1);
        wv[k][c] = s;
      }
    }
    const float mk = r[4];
    for (int c = 0; c < 3; ++c) {
      const float v = mk * wv[0][c] + (1.f - mk) * wv[1][c] + m + r[5 + c];
      out[(size_t)c * H * W + i] = fminf(fmaxf(v, 0.f), 1.f);
    }
  }
}

}  // namespace

int ifrnet_sum_blocks() { return 256; }

cudaError_t launch_ifrnet_mean(const float* f0, const float* f1, int H, int W, int Hp, int Wp, double* partial, float* mean,
                               cudaStream_t st) {
  const int nb = ifrnet_sum_blocks();
  cudaMemsetAsync(partial, 0, sizeof(double) * nb, st);
  VFI_LAUNCH(ifr_frame_sums_kernel, nb, 256, 0, st, f0, f1, (size_t)3 * H * W, partial);
  VFI_LAUNCH(ifr_mean_kernel, 1, 32, 0, st, partial, nb, 6.0 * Hp * Wp, mean);
  return cudaGetLastError();
}

cudaError_t launch_ifrnet_prep(const float* f0, const float* f1, int H, int W, int Hp, int Wp, int h0, int w0, float scale,
                               const float* mean, float4* out, cudaStream_t st) {
  VFI_LAUNCH(ifr_prep_kernel, ifr_grid((size_t)2 * h0 * w0, 256), 256, 0, st, f0, f1, H, W, Hp, Wp, h0, w0, scale, mean, out);
  return cudaGetLastError();
}

cudaError_t launch_ifrnet_first_conv(int op, const float4* xin, int h0, int w0, int h1, int w1, int k, const float* w,
                                     const float* bias, const float* slopes, int C, int pitch, void* out, cudaStream_t st) {
  const int g = ifr_grid((size_t)2 * h1 * w1 * (pitch / 8), 128);
  if (op == OP_BF16)
    VFI_LAUNCH(ifr_first_conv_kernel<__nv_bfloat16>, g, 128, 0, st, xin, h0, w0, h1, w1, k, w, bias, slopes, C, pitch,
               (__nv_bfloat16*)out);
  else
    VFI_LAUNCH(ifr_first_conv_kernel<__half>, g, 128, 0, st, xin, h0, w0, h1, w1, k, w, bias, slopes, C, pitch, (__half*)out);
  return cudaGetLastError();
}

cudaError_t launch_ifrnet_s2d(int op, const void* in, int pitch, int cq, int B, int h, int w, void* out, int opitch,
                              cudaStream_t st) {
  const int g = ifr_grid((size_t)B * ((h + 1) / 2) * ((w + 1) / 2) * (opitch / 8), 256);
  if (op == OP_BF16)
    VFI_LAUNCH(ifr_s2d_kernel<__nv_bfloat16>, g, 256, 0, st, (const __nv_bfloat16*)in, pitch, cq, B, h, w,
               (__nv_bfloat16*)out, opitch);
  else
    VFI_LAUNCH(ifr_s2d_kernel<__half>, g, 256, 0, st, (const __half*)in, pitch, cq, B, h, w, (__half*)out, opitch);
  return cudaGetLastError();
}

cudaError_t launch_ifrnet_dec4_in(int op, const void* f, int fpitch, int g1, int h, int w, float embt, void* out,
                                  cudaStream_t st) {
  const int g = ifr_grid((size_t)h * w * ((2 * g1 + 64) / 8), 256);
  if (op == OP_BF16)
    VFI_LAUNCH(ifr_dec4_in_kernel<__nv_bfloat16>, g, 256, 0, st, (const __nv_bfloat16*)f, fpitch, g1, h, w, embt,
               (__nv_bfloat16*)out);
  else
    VFI_LAUNCH(ifr_dec4_in_kernel<__half>, g, 256, 0, st, (const __half*)f, fpitch, g1, h, w, embt, (__half*)out);
  return cudaGetLastError();
}

cudaError_t launch_ifrnet_dec_flow(const float* ph, int nf, const float* prev, int h, int w, float* acc, cudaStream_t st) {
  VFI_LAUNCH(ifr_dec_flow_kernel, ifr_grid((size_t)4 * h * w, 256), 256, 0, st, ph, nf, prev, h, w, acc);
  return cudaGetLastError();
}

cudaError_t launch_ifrnet_dec_in(int op, const void* ph16, int pp, const void* f, int fpitch, int fh, int fw,
                                 const float* acc, int gh, int gw, int g1, int g2, int g3, void* out, cudaStream_t st) {
  const int g = ifr_grid((size_t)gh * gw * ((g3 + 64) / 8), 256);
  if (op == OP_BF16)
    VFI_LAUNCH(ifr_dec_in_kernel<__nv_bfloat16>, g, 256, 0, st, (const __nv_bfloat16*)ph16, pp, (const __nv_bfloat16*)f,
               fpitch, fh, fw, acc, gh, gw, g1, g2, g3, (__nv_bfloat16*)out);
  else
    VFI_LAUNCH(ifr_dec_in_kernel<__half>, g, 256, 0, st, (const __half*)ph16, pp, (const __half*)f, fpitch, fh, fw, acc, gh,
               gw, g1, g2, g3, (__half*)out);
  return cudaGetLastError();
}

cudaError_t launch_ifrnet_final(const float* f0, const float* f1, int H, int W, int Hp, int Wp, const float* acc, int hq,
                                int wq, int hF, int wF, float scale, float fmul, const float* mean, float* out,
                                cudaStream_t st) {
  VFI_LAUNCH(ifr_final_kernel, ifr_grid((size_t)H * W, 256), 256, 0, st, f0, f1, H, W, Hp, Wp, acc, hq, wq, hF, wF, scale,
             fmul, mean, out);
  return cudaGetLastError();
}

}  // namespace vfi
