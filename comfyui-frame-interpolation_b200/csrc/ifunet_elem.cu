// The kernels of the IFUnet path (ifunet.cu) around its tensor-core convolutions, on the CUDA cores.
// Activations are 16-bit NHWC tensors; flows, masks, gates, warps and the blends are fp32.  Frames and the output are
// fp32 [3][H][W] planes; every padded frame (Hp x Wp) reads them with zeros beyond H x W.
// Reference: vfi_models/ifunet/IFUNet_arch.py.
//
//   flow_in      IFUNet level input: cat(a, b, t[, warped0, warped1]) (resized by scale), [+ flow], the 7 -> 17
//                conv0 + PReLU at level 0; written as the space-to-depth copy FeatureNet.conv1.conv1 reads
//   s2d          the space-to-depth copy every other stride-2 conv reads as a 2x2 conv
//   d2s          the four ConvTranspose2d(4, 2, 1) phase outputs interleaved onto the doubled grid
//   pool, gate   CBAM channel gate: fixed-order partial sums / maxima per image, the shared MLP on both, sigmoid
//   compress     CBAM ChannelPool of x * gate: per-pixel channel max and mean (fp32)
//   spatial      CBAM spatial gate (7x7 conv 2 -> 1 with BatchNorm folded, sigmoid) and out = (x * gate) * s
//   add16        x += y, the residual of convblock(x) + x (after the last PReLU)
//   convex       IFBlock.upsample_flow: softmax over the 9 taps of the mask, applied to unfold(level * flow)
//   flow_update  F.interpolate(flow_up, 1 / scale) * (1 / scale), the ensemble average and the flow accumulation
//   warp_frames  warp(img0, flow[:2]), warp(img1, flow[2:4]) on the padded frames
//   fusion_in    RRDBNet input: cat(img0, img1, w0, w1) resized by 1/4, flow resized by 1/4 times 1/4
//   rrdb_res     RRDB: out * 0.2 + x
//   merge        sigmoid(conv_last) blend of the warped frames: the `deg` image
//   fb_in        FlowBlock input: cat(img, deg[, warped, mask]) resized by 1 / scale[, flow resized times 1 / scale]
//   stem         3x3 stride-2 conv on a few fp32 planes + per-channel affine + PReLU (conv_bn / context stems)
//   fb_out       FlowBlock tail: the ConvT phases resized by 4 scale, flow * 4 scale, mask; accumulated; warp(img, flow)
//   ctx_warp     warp(context0(img), F.interpolate(flow, 0.25) * 0.25) into channels [0, 32) of the decode input
//   final        tanh of decode, + warped, clamp, softmax(clamp(m0, m1, 0)) blend with deg, crop
#include "ptx.cuh"
#include "vfi_internal.h"

namespace vfi {

namespace {

inline int ifu_grid(size_t total, int threads) {
  size_t b = (total + threads - 1) / threads;
  return (int)(b < 1 ? 1 : (b > 1048576 ? 1048576 : b));
}

template <typename T>
__device__ __forceinline__ void ifu_ld8(const T* p, float (&f)[8]) {
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
__device__ __forceinline__ void ifu_st8(T* p, const float (&f)[8]) {
  uint4 u;
  u.x = Pack2<T>::pack(f[0], f[1]);
  u.y = Pack2<T>::pack(f[2], f[3]);
  u.z = Pack2<T>::pack(f[4], f[5]);
  u.w = Pack2<T>::pack(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// F.interpolate(bilinear, align_corners=False) source index along one axis: src = scale * (dst + 0.5) - 0.5 with the
// fp32 coordinate scale (1 / scale_factor), clamped at 0; i1 = i0 + 1 unless i0 is the last row
struct Lin {
  int i0, i1;
  float l0, l1;
};
__device__ __forceinline__ Lin ifu_lin(float scale, int dst, int in_size) {
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
// identity when the grid is not resized (F.interpolate with scale_factor 1.0 copies)
__device__ __forceinline__ Lin ifu_lin_or_id(bool resize, float scale, int dst, int in_size) {
  if (resize) return ifu_lin(scale, dst, in_size);
  Lin r;
  r.i0 = r.i1 = dst;
  r.l0 = 1.f;
  r.l1 = 0.f;
  return r;
}

// torch.linspace(-1, 1, n)[i] in fp32
__device__ __forceinline__ float ifu_linspace(int i, int n) {
  const float step = 2.0f / (float)(n - 1);
  return i < n / 2 ? -1.f + step * (float)i : 1.f - step * (float)(n - 1 - i);
}

// warp(): grid from the flow's size (gw x gh), grid_sample(bilinear, border, align_corners=True) of an image of its own
// size (iw x ih); the four corner indices (-1: outside, weight skipped) and weights
struct Tap4 {
  int x0, y0, x1, y1;
  float w00, w01, w10, w11;
};
__device__ __forceinline__ Tap4 ifu_warp_taps(int X, int Y, int gw, int gh, float fx, float fy, int iw, int ih) {
  const float gx = ifu_linspace(X, gw) + fx / (((float)iw - 1.0f) / 2.0f);
  const float gy = ifu_linspace(Y, gh) + fy / (((float)ih - 1.0f) / 2.0f);
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

// a plane of the padded frame: zero beyond the H x W frame
__device__ __forceinline__ float ifu_px(const float* pl, int H, int W, int y, int x) {
  return (y < H && x < W) ? pl[(size_t)y * W + x] : 0.f;
}

__device__ __forceinline__ float ifu_warp_plane(const float* pl, int H, int W, const Tap4& t) {
  float s = 0.f;
  if (t.y0 >= 0 && t.x0 >= 0) s += t.w00 * ifu_px(pl, H, W, t.y0, t.x0);
  if (t.y0 >= 0 && t.x1 >= 0) s += t.w01 * ifu_px(pl, H, W, t.y0, t.x1);
  if (t.y1 >= 0 && t.x0 >= 0) s += t.w10 * ifu_px(pl, H, W, t.y1, t.x0);
  if (t.y1 >= 0 && t.x1 >= 0) s += t.w11 * ifu_px(pl, H, W, t.y1, t.x1);
  return s;
}

template <class F>
__device__ __forceinline__ float ifu_bilin(const Lin& ly, const Lin& lx, F at) {
  return ly.l0 * (lx.l0 * at(ly.i0, lx.i0) + lx.l1 * at(ly.i0, lx.i1)) +
         ly.l1 * (lx.l0 * at(ly.i1, lx.i0) + lx.l1 * at(ly.i1, lx.i1));
}

// ---------------------------------------------------------------- IFUNet level input
// One item = (pixel of the ceil(h0/2) x ceil(w0/2) grid, phase q): the 17 channels of input pixel (2Y + py, 2X + px) at
// q * 24 (zero outside the input and in [17, 24)); q = 3 also zeroes [96, 128).  Images b of a batch: b = 1 is the
// ensemble pass, cat(img1, img0, 1 - t, ...).

template <typename T>
__global__ void ifu_flow_in_kernel(const IfuFlowIn a, int B, T* __restrict__ out) {
  const int ho = (a.h0 + 1) / 2, wo = (a.w0 + 1) / 2;
  const size_t total = (size_t)B * ho * wo * 4;
  const size_t plane = (size_t)a.Hp * a.Wp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = (int)(i & 3);
    const size_t pix = i >> 2;
    const int X = (int)(pix % wo), Y = (int)((pix / wo) % ho), b = (int)(pix / ((size_t)wo * ho));
    const int y = 2 * Y + (q >> 1), x = 2 * X + (q & 1);
    float v[24];
#pragma unroll
    for (int c = 0; c < 24; ++c) v[c] = 0.f;
    if (y < a.h0 && x < a.w0) {
      const bool sw = (b == 1) != (a.swap0 != 0);
      const float* ia = sw ? a.f1 : a.f0;
      const float* ib = sw ? a.f0 : a.f1;
      const float tt = sw ? 1.f - a.t : a.t;
      const Lin ly = ifu_lin_or_id(a.resize, a.cscale, y, a.Hp), lx = ifu_lin_or_id(a.resize, a.cscale, x, a.Wp);
      float in[17];
      for (int c = 0; c < 3; ++c) {
        const float* pa = ia + (size_t)c * a.H * a.W;
        const float* pb = ib + (size_t)c * a.H * a.W;
        in[c] = ifu_bilin(ly, lx, [&](int yy, int xx) { return ifu_px(pa, a.H, a.W, yy, xx); });
        in[3 + c] = ifu_bilin(ly, lx, [&](int yy, int xx) { return ifu_px(pb, a.H, a.W, yy, xx); });
      }
      in[6] = ifu_bilin(ly, lx, [&](int, int) { return tt; });
      if (a.warped) {
        for (int c = 0; c < 6; ++c) {
          const float* pw = a.warped + c * plane;
          in[7 + c] = ifu_bilin(ly, lx, [&](int yy, int xx) { return pw[(size_t)yy * a.Wp + xx]; });
        }
        for (int c = 0; c < 4; ++c) {
          const float f = ifu_bilin(ly, lx, [&](int yy, int xx) { return a.flow[((size_t)yy * a.Wp + xx) * 4 + c]; });
          in[13 + c] = a.resize ? f * a.fscale : f;
        }
        for (int c = 0; c < 17; ++c) v[c] = in[c];
      } else {
        for (int o = 0; o < 17; ++o) {
          float s = a.c0b[o];
          for (int c = 0; c < 7; ++c) s = fmaf(a.c0w[o * 7 + c], in[c], s);
          v[o] = s > 0.f ? s : a.c0s[o] * s;
        }
      }
    }
    T* o = out + pix * 128 + q * 24;
    ifu_st8(o, *reinterpret_cast<float(*)[8]>(v));
    ifu_st8(o + 8, *reinterpret_cast<float(*)[8]>(v + 8));
    ifu_st8(o + 16, *reinterpret_cast<float(*)[8]>(v + 16));
    if (q == 3) {
      const float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int k = 0; k < 4; ++k) ifu_st8(out + pix * 128 + 96 + 8 * k, z);
    }
  }
}

// space-to-depth: out[b][Y][X][q * cq + c] = in[b][2Y + py][2X + px][c] (c < cq), zero outside the input and in
// [4 cq, opitch)
template <typename T>
__global__ void ifu_s2d_kernel(const T* __restrict__ in, int pitch, int cq, int B, int h, int w, T* __restrict__ out,
                               int opitch) {
  const int ho = (h + 1) / 2, wo = (w + 1) / 2, chunks = opitch / 8, qc = cq / 8;
  const size_t total = (size_t)B * ho * wo * chunks;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % chunks);
    const size_t pix = i / chunks;
    const int X = (int)(pix % wo), Y = (int)((pix / wo) % ho), b = (int)(pix / ((size_t)wo * ho));
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    const int q = ch / qc;
    if (q < 4) {
      const int y = 2 * Y + (q >> 1), x = 2 * X + (q & 1);
      if (y < h && x < w) v = *reinterpret_cast<const uint4*>(in + (((size_t)b * h + y) * w + x) * pitch + (ch - q * qc) * 8);
    }
    *reinterpret_cast<uint4*>(out + pix * opitch + ch * 8) = v;
  }
}

// ConvT phases ph [4][B][h][w][C] (phase q = py * 2 + px) -> out [B][2h][2w][C]
__global__ void ifu_d2s_kernel(const uint4* __restrict__ ph, int C8, int B, int h, int w, uint4* __restrict__ out) {
  const size_t total = (size_t)B * 4 * h * w * C8;
  const size_t pl = (size_t)B * h * w * C8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C8);
    const size_t px = i / C8;
    const int X = (int)(px % (2 * w)), Y = (int)((px / (2 * w)) % (2 * h)), b = (int)(px / ((size_t)4 * h * w));
    const int q = (Y & 1) * 2 + (X & 1);
    out[i] = ph[q * pl + (((size_t)b * h + (Y >> 1)) * w + (X >> 1)) * C8 + c];
  }
}

// ---------------------------------------------------------------- CBAM
// partial sums / maxima of chunk k of image b: [B][kIfuPoolChunks][C]; a block per chunk (grid-stride) and image
// (blockIdx.y), kPoolLanes pixel lanes x 8-channel vectors, the lanes combined in a fixed order
constexpr int kPoolLanes = 4;
template <typename T>
__global__ void ifu_pool_kernel(const T* __restrict__ x, int pitch, int C, int npx, float* __restrict__ psum,
                                float* __restrict__ pmax) {
  __shared__ float red[kPoolLanes][2][512];
  const int b = blockIdx.y, C8 = C / 8;
  const int len = (npx + kIfuPoolChunks - 1) / kIfuPoolChunks;
  for (int k = blockIdx.x; k < kIfuPoolChunks; k += gridDim.x) {
    const int p0 = k * len, p1 = min(npx, p0 + len);
    for (int it = threadIdx.x; it < kPoolLanes * C8; it += blockDim.x) {
      const int lane = it / C8, v = it - lane * C8;
      float s[8], m[8];
      for (int j = 0; j < 8; ++j) {
        s[j] = 0.f;
        m[j] = -INFINITY;
      }
      for (int p = p0 + lane; p < p1; p += kPoolLanes) {
        float f[8];
        ifu_ld8(x + ((size_t)b * npx + p) * pitch + v * 8, f);
        for (int j = 0; j < 8; ++j) {
          s[j] += f[j];
          m[j] = fmaxf(m[j], f[j]);
        }
      }
      for (int j = 0; j < 8; ++j) {
        red[lane][0][v * 8 + j] = s[j];
        red[lane][1][v * 8 + j] = m[j];
      }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      float s = 0.f, m = -INFINITY;
      for (int l = 0; l < kPoolLanes; ++l) {
        s += red[l][0][c];
        m = fmaxf(m, red[l][1][c]);
      }
      psum[((size_t)b * kIfuPoolChunks + k) * C + c] = s;
      pmax[((size_t)b * kIfuPoolChunks + k) * C + c] = m;
    }
    __syncthreads();
  }
}

// g[b][c] = sigmoid(mlp(avg) + mlp(max)), mlp(v) = W2 relu(W1 v + b1) + b2; mlp = {W1 [hid][C], b1, W2 [C][hid], b2};
// a block per image (grid-stride)
__global__ void ifu_gate_kernel(const float* __restrict__ psum, const float* __restrict__ pmax, int C, int hid, int npx,
                                int B, const float* __restrict__ mlp, float* __restrict__ g) {
  __shared__ float avg[512], mx[512], hd[64];
  const float* w1 = mlp;
  const float* b1 = w1 + hid * C;
  const float* w2 = b1 + hid;
  const float* b2 = w2 + C * hid;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      float s = 0.f, m = -INFINITY;
      for (int k = 0; k < kIfuPoolChunks; ++k) {
        s += psum[((size_t)b * kIfuPoolChunks + k) * C + c];
        m = fmaxf(m, pmax[((size_t)b * kIfuPoolChunks + k) * C + c]);
      }
      avg[c] = s / (float)npx;
      mx[c] = m;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < 2 * hid; j += blockDim.x) {
      const float* v = j < hid ? avg : mx;
      const int r = j % hid;
      float a = b1[r];
      for (int c = 0; c < C; ++c) a = fmaf(w1[r * C + c], v[c], a);
      hd[j] = fmaxf(a, 0.f);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      float a0 = b2[c], a1 = b2[c];
      for (int r = 0; r < hid; ++r) {
        a0 = fmaf(w2[c * hid + r], hd[r], a0);
        a1 = fmaf(w2[c * hid + r], hd[hid + r], a1);
      }
      g[(size_t)b * C + c] = 1.f / (1.f + expf(-(a0 + a1)));
    }
    __syncthreads();
  }
}

// cmp[b][p] = {max_c x * g, mean_c x * g}
template <typename T>
__global__ void ifu_compress_kernel(const T* __restrict__ x, int pitch, int C, int B, int npx, const float* __restrict__ g,
                                    float2* __restrict__ cmp) {
  const size_t total = (size_t)B * npx;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / npx);
    const float* gb = g + (size_t)b * C;
    float m = -INFINITY, s = 0.f;
    for (int c0 = 0; c0 < C; c0 += 8) {
      float f[8];
      ifu_ld8(x + i * pitch + c0, f);
      for (int j = 0; j < 8; ++j) {
        const float y = f[j] * gb[c0 + j];
        m = fmaxf(m, y);
        s += y;
      }
    }
    cmp[i] = make_float2(m, s / (float)C);
  }
}

// out = (x * g) * sigmoid(conv7x7(cmp) + bias); sw = {w [2][7][7] (BatchNorm folded), bias}; in place allowed
template <typename T>
__global__ void ifu_spatial_kernel(const T* __restrict__ x, int pitch, int C, int B, int h, int w,
                                   const float* __restrict__ g, const float2* __restrict__ cmp, const float* __restrict__ sw,
                                   T* __restrict__ out) {
  const int C8 = C / 8;
  const size_t total = (size_t)B * h * w * C8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % C8);
    const size_t pix = i / C8;
    const int X = (int)(pix % w), Y = (int)((pix / w) % h), b = (int)(pix / ((size_t)w * h));
    float s = sw[98];
    for (int ky = 0; ky < 7; ++ky) {
      const int yy = Y + ky - 3;
      if (yy < 0 || yy >= h) continue;
      for (int kx = 0; kx < 7; ++kx) {
        const int xx = X + kx - 3;
        if (xx < 0 || xx >= w) continue;
        const float2 c = cmp[((size_t)b * h + yy) * w + xx];
        s = fmaf(sw[ky * 7 + kx], c.x, s);
        s = fmaf(sw[49 + ky * 7 + kx], c.y, s);
      }
    }
    const float sg = 1.f / (1.f + expf(-s));
    float f[8];
    ifu_ld8(x + pix * pitch + v * 8, f);
    const float* gb = g + (size_t)b * C + v * 8;
    for (int j = 0; j < 8; ++j) f[j] = (f[j] * gb[j]) * sg;
    ifu_st8(out + pix * pitch + v * 8, f);
  }
}

// x += y over n 8-element vectors
template <typename T>
__global__ void ifu_add_kernel(T* __restrict__ x, const T* __restrict__ y, size_t n8) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (size_t)gridDim.x * blockDim.x) {
    float a[8], b[8];
    ifu_ld8(x + i * 8, a);
    ifu_ld8(y + i * 8, b);
    for (int j = 0; j < 8; ++j) a[j] += b[j];
    ifu_st8(x + i * 8, a);
  }
}

// ---------------------------------------------------------------- IFBlock tail
// up[b][Y][X][k] on the (L h) x (L w) grid, Y = y L + a, X = x L + c: sum_t softmax_t(mask[b][y][x][t L L + a L + c]) *
// L * flow[b][y + t / 3 - 1][x + t % 3 - 1][k] (zero outside)
template <typename T>
__global__ void ifu_convex_kernel(const float* __restrict__ flow, const T* __restrict__ mask, int L, int B, int h, int w,
                                  float* __restrict__ up) {
  const int H = L * h, W = L * w, LL = L * L;
  const size_t total = (size_t)B * H * W;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int X = (int)(i % W), Y = (int)((i / W) % H), b = (int)(i / ((size_t)W * H));
    const int y = Y / L, a = Y - y * L, x = X / L, c = X - x * L;
    const size_t cell = ((size_t)b * h + y) * w + x;
    const T* mk = mask + cell * (9 * LL) + a * L + c;
    float lg[9], mx = -INFINITY;
    for (int t = 0; t < 9; ++t) {
      lg[t] = (float)mk[t * LL];
      mx = fmaxf(mx, lg[t]);
    }
    float den = 0.f;
    for (int t = 0; t < 9; ++t) {
      lg[t] = expf(lg[t] - mx);
      den += lg[t];
    }
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int t = 0; t < 9; ++t) {
      const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
      if (yy < 0 || yy >= h || xx < 0 || xx >= w) continue;
      const float p = lg[t] / den;
      const float* f = flow + (((size_t)b * h + yy) * w + xx) * 4;
      for (int k = 0; k < 4; ++k) acc[k] += p * ((float)L * f[k]);
    }
    reinterpret_cast<float4*>(up)[i] = make_float4(acc[0], acc[1], acc[2], acc[3]);
  }
}

// d_b = resize(up_b, 1 / scale) * (1 / scale) at Hp x Wp (a copy at scale 1); flow = mode 0: d_0, 1: (d_0 + d_1) / 2,
// 2: flow + d_0, 3: (flow + (flow + d_0)) / 2
__global__ void ifu_flow_update_kernel(const float4* __restrict__ up, int uh, int uw, int resize, float cscale, float fmul,
                                       int mode, int Hp, int Wp, float4* __restrict__ flow) {
  const size_t total = (size_t)Hp * Wp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int X = (int)(i % Wp), Y = (int)(i / Wp);
    const Lin ly = ifu_lin_or_id(resize, cscale, Y, uh), lx = ifu_lin_or_id(resize, cscale, X, uw);
    float d[2][4];
    for (int b = 0; b < (mode == 1 ? 2 : 1); ++b) {
      const float4* u = up + (size_t)b * uh * uw;
      for (int k = 0; k < 4; ++k) {
        const float v = ifu_bilin(ly, lx, [&](int yy, int xx) {
          const float4 q = u[(size_t)yy * uw + xx];
          return k == 0 ? q.x : (k == 1 ? q.y : (k == 2 ? q.z : q.w));
        });
        d[b][k] = v * fmul;
      }
    }
    float o[4];
    if (mode == 0) {
      for (int k = 0; k < 4; ++k) o[k] = d[0][k];
    } else if (mode == 1) {
      for (int k = 0; k < 4; ++k) o[k] = (d[0][k] + d[1][k]) / 2.f;
    } else {
      const float4 f = flow[i];
      const float fb[4] = {f.x, f.y, f.z, f.w};
      for (int k = 0; k < 4; ++k) o[k] = mode == 2 ? fb[k] + d[0][k] : (fb[k] + (fb[k] + d[0][k])) / 2.f;
    }
    flow[i] = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// warped[k][c] = warp(img_k, flow[2k : 2k + 2]) on the padded frames
__global__ void ifu_warp_frames_kernel(const float* __restrict__ f0, const float* __restrict__ f1, int H, int W, int Hp,
                                       int Wp, const float4* __restrict__ flow, float* __restrict__ warped) {
  const size_t plane = (size_t)Hp * Wp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < plane; i += (size_t)gridDim.x * blockDim.x) {
    const int X = (int)(i % Wp), Y = (int)(i / Wp);
    const float4 f = flow[i];
    for (int k = 0; k < 2; ++k) {
      const Tap4 t = ifu_warp_taps(X, Y, Wp, Hp, k ? f.z : f.x, k ? f.w : f.y, Wp, Hp);
      const float* img = k ? f1 : f0;
      for (int c = 0; c < 3; ++c) warped[(k * 3 + c) * plane + i] = ifu_warp_plane(img + (size_t)c * H * W, H, W, t);
    }
  }
}

// ---------------------------------------------------------------- fusion (RRDBNet)
// out[y][x][0..16) = cat(img0, img1, w0, w1) resized by 1/4, flow resized by 1/4 times 0.25; [16, 64) zero
template <typename T>
__global__ void ifu_fusion_in_kernel(const float* __restrict__ f0, const float* __restrict__ f1, int H, int W, int Hp,
                                     int Wp, const float* __restrict__ warped, const float4* __restrict__ flow,
                                     T* __restrict__ out) {
  const int hq = Hp / 4, wq = Wp / 4;
  const size_t total = (size_t)hq * wq, plane = (size_t)Hp * Wp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % wq), y = (int)(i / wq);
    const Lin ly = ifu_lin(4.f, y, Hp), lx = ifu_lin(4.f, x, Wp);
    float v[64];
    for (int c = 0; c < 64; ++c) v[c] = 0.f;
    for (int c = 0; c < 3; ++c) {
      const float* p0 = f0 + (size_t)c * H * W;
      const float* p1 = f1 + (size_t)c * H * W;
      v[c] = ifu_bilin(ly, lx, [&](int yy, int xx) { return ifu_px(p0, H, W, yy, xx); });
      v[3 + c] = ifu_bilin(ly, lx, [&](int yy, int xx) { return ifu_px(p1, H, W, yy, xx); });
    }
    for (int c = 0; c < 6; ++c) {
      const float* pw = warped + c * plane;
      v[6 + c] = ifu_bilin(ly, lx, [&](int yy, int xx) { return pw[(size_t)yy * Wp + xx]; });
    }
    for (int k = 0; k < 4; ++k)
      v[12 + k] = ifu_bilin(ly, lx, [&](int yy, int xx) {
                    const float4 q = flow[(size_t)yy * Wp + xx];
                    return k == 0 ? q.x : (k == 1 ? q.y : (k == 2 ? q.z : q.w));
                  }) * 0.25f;
    for (int c = 0; c < 64; c += 8) ifu_st8(out + i * 64 + c, *reinterpret_cast<float(*)[8]>(v + c));
  }
}

// y = y * 0.2 + x over n 8-element vectors
template <typename T>
__global__ void ifu_rrdb_res_kernel(T* __restrict__ y, const T* __restrict__ x, size_t n8) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (size_t)gridDim.x * blockDim.x) {
    float a[8], b[8];
    ifu_ld8(y + i * 8, a);
    ifu_ld8(x + i * 8, b);
    for (int j = 0; j < 8; ++j) a[j] = a[j] * 0.2f + b[j];
    ifu_st8(y + i * 8, a);
  }
}

// deg[c] = w0 * m + w1 * (1 - m), m = sigmoid(conv_last) (fp32 [Hp][Wp][2], column 0)
__global__ void ifu_merge_kernel(const float* __restrict__ warped, const float* __restrict__ last, int Hp, int Wp,
                                 float* __restrict__ deg) {
  const size_t plane = (size_t)Hp * Wp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < plane; i += (size_t)gridDim.x * blockDim.x) {
    const float m = 1.f / (1.f + expf(-last[i * 2]));
    for (int c = 0; c < 3; ++c) deg[c * plane + i] = warped[c * plane + i] * m + warped[(3 + c) * plane + i] * (1.f - m);
  }
}

// ---------------------------------------------------------------- ResynNet
// FlowBlock input of image b (0: img0, 1: img1) as fp32 planes [2][cin][h][w], h = Hp / s (a copy at s = 1): cat(img,
// deg) (cin 6), or cat(img, deg, warped, mask) resized + flow resized / s (cin 12)
__global__ void ifu_fb_in_kernel(const float* __restrict__ f0, const float* __restrict__ f1, int H, int W, int Hp, int Wp,
                                 const float* __restrict__ deg, const float* __restrict__ rwarp,
                                 const float* __restrict__ rmask, const float2* __restrict__ rflow, int cin, int s,
                                 float* __restrict__ out) {
  const int h = Hp / s, w = Wp / s;
  const size_t hw = (size_t)h * w, total = 2 * hw, plane = (size_t)Hp * Wp;
  const float cs = (float)s, inv = (float)s;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / hw);
    const size_t p = i - b * hw;
    const int x = (int)(p % w), y = (int)(p / w);
    const Lin ly = ifu_lin_or_id(s != 1, cs, y, Hp), lx = ifu_lin_or_id(s != 1, cs, x, Wp);
    float* o = out + (size_t)b * cin * hw + p;
    const float* img = b ? f1 : f0;
    for (int c = 0; c < 3; ++c) {
      const float* pi = img + (size_t)c * H * W;
      const float* pd = deg + c * plane;
      o[c * hw] = ifu_bilin(ly, lx, [&](int yy, int xx) { return ifu_px(pi, H, W, yy, xx); });
      o[(3 + c) * hw] = ifu_bilin(ly, lx, [&](int yy, int xx) { return pd[(size_t)yy * Wp + xx]; });
    }
    if (cin == 12) {
      for (int c = 0; c < 3; ++c) {
        const float* pw = rwarp + (b * 3 + c) * plane;
        o[(6 + c) * hw] = ifu_bilin(ly, lx, [&](int yy, int xx) { return pw[(size_t)yy * Wp + xx]; });
      }
      const float* pm = rmask + b * plane;
      o[9 * hw] = ifu_bilin(ly, lx, [&](int yy, int xx) { return pm[(size_t)yy * Wp + xx]; });
      const float2* pf = rflow + b * plane;
      for (int k = 0; k < 2; ++k)
        o[(10 + k) * hw] = ifu_bilin(ly, lx, [&](int yy, int xx) {
                             const float2 q = pf[(size_t)yy * Wp + xx];
                             return k ? q.y : q.x;
                           }) * 1.0f / inv;
    }
  }
}

// 3x3 stride-2 conv (padding 1) over an sh x sw grid of image b's fp32 planes src[b] [cin][vh][vw] (zero beyond them),
// + bias, PReLU ->
// 16-bit [B][ho][wo][pitch]; channels [cout, pitch) zero.  w [cout][cin][9] (BatchNorm folded).
struct StemSrc {
  const float* p[2];
};
template <typename T>
__global__ void ifu_stem_kernel(StemSrc src, int cin, int sh, int sw, int vh, int vw, const float* __restrict__ w,
                                const float* __restrict__ bias, const float* __restrict__ slopes, int cout, int B, int ho,
                                int wo, int pitch, T* __restrict__ out) {
  const int chunks = pitch / 8;
  const size_t total = (size_t)B * ho * wo * chunks;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % chunks);
    const size_t pix = i / chunks;
    const int ox = (int)(pix % wo), oy = (int)((pix / wo) % ho), b = (int)(pix / ((size_t)wo * ho));
    float acc[8];
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    const int c0 = ch * 8;
    if (c0 < cout) {
      for (int j = 0; j < 8; ++j) acc[j] = c0 + j < cout ? bias[c0 + j] : 0.f;
      const float* s = src.p[b];
      for (int ky = 0; ky < 3; ++ky) {
        const int y = 2 * oy + ky - 1;
        if (y < 0 || y >= sh) continue;
        for (int kx = 0; kx < 3; ++kx) {
          const int x = 2 * ox + kx - 1;
          if (x < 0 || x >= sw) continue;
          for (int c = 0; c < cin; ++c) {
            const float v = (y < vh && x < vw) ? s[((size_t)c * vh + y) * vw + x] : 0.f;
            for (int j = 0; j < 8; ++j)
              if (c0 + j < cout) acc[j] = fmaf(v, w[((size_t)(c0 + j) * cin + c) * 9 + ky * 3 + kx], acc[j]);
          }
        }
      }
      for (int j = 0; j < 8; ++j)
        if (c0 + j < cout) acc[j] = acc[j] > 0.f ? acc[j] : slopes[c0 + j] * acc[j];
    }
    ifu_st8(out + pix * pitch + c0, acc);
  }
}

// FlowBlock tail: tmp = resize(ConvT phases, 4 s) at Hp x Wp (ph [4][2][h][w][4], the ConvT grid 2h x 2w), flow =
// tmp[:2] * s * 4, mask = tmp[2]; accumulated unless first; rwarp = warp(img_b, flow)
__global__ void ifu_fb_out_kernel(const float* __restrict__ ph, int h, int w, int s, int first, const float* __restrict__ f0,
                                  const float* __restrict__ f1, int H, int W, int Hp, int Wp, float2* __restrict__ rflow,
                                  float* __restrict__ rmask, float* __restrict__ rwarp) {
  const size_t plane = (size_t)Hp * Wp, total = 2 * plane;
  const size_t pl = (size_t)2 * h * w * 4;
  const float cs = (float)(1.0 / (4.0 * s)), fs = (float)s;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / plane);
    const size_t p = i - b * plane;
    const int X = (int)(p % Wp), Y = (int)(p / Wp);
    const Lin ly = ifu_lin(cs, Y, 2 * h), lx = ifu_lin(cs, X, 2 * w);
    float v[3];
    for (int c = 0; c < 3; ++c)
      v[c] = ifu_bilin(ly, lx, [&](int yy, int xx) {
        const int q = (yy & 1) * 2 + (xx & 1);
        return ph[q * pl + (((size_t)b * h + (yy >> 1)) * w + (xx >> 1)) * 4 + c];
      });
    float2 fl = make_float2(v[0] * fs * 4.f, v[1] * fs * 4.f);
    float m = v[2];
    if (!first) {
      const float2 o = rflow[i];
      fl = make_float2(o.x + fl.x, o.y + fl.y);
      m = rmask[i] + m;
    }
    rflow[i] = fl;
    rmask[i] = m;
    const Tap4 t = ifu_warp_taps(X, Y, Wp, Hp, fl.x, fl.y, Wp, Hp);
    const float* img = b ? f1 : f0;
    for (int c = 0; c < 3; ++c) rwarp[(b * 3 + c) * plane + p] = ifu_warp_plane(img + (size_t)c * H * W, H, W, t);
  }
}

// out[b][y][x][0..32) (pitch 64) = warp(feat[b] (h x w, pitch fpitch), resize(rflow[b], 0.25) * 0.25), h = Hp / 4
template <typename T>
__global__ void ifu_ctx_warp_kernel(const T* __restrict__ feat, int fpitch, const float2* __restrict__ rflow, int Hp,
                                    int Wp, T* __restrict__ out) {
  const int h = Hp / 4, w = Wp / 4;
  const size_t total = (size_t)2 * h * w * 4, plane = (size_t)Hp * Wp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int v = (int)(i & 3);
    const size_t pix = i >> 2;
    const int x = (int)(pix % w), y = (int)((pix / w) % h), b = (int)(pix / ((size_t)w * h));
    const Lin ly = ifu_lin(4.f, y, Hp), lx = ifu_lin(4.f, x, Wp);
    const float2* pf = rflow + b * plane;
    const float fx = ifu_bilin(ly, lx, [&](int yy, int xx) { return pf[(size_t)yy * Wp + xx].x; }) * 0.25f;
    const float fy = ifu_bilin(ly, lx, [&](int yy, int xx) { return pf[(size_t)yy * Wp + xx].y; }) * 0.25f;
    const Tap4 t = ifu_warp_taps(x, y, w, h, fx, fy, w, h);
    const T* src = feat + (size_t)b * h * w * fpitch + v * 8;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, q[8];
    auto add = [&](int yy, int xx, float wt) {
      if (yy < 0 || xx < 0) return;
      ifu_ld8(src + ((size_t)yy * w + xx) * fpitch, q);
      for (int j = 0; j < 8; ++j) acc[j] += wt * q[j];
    };
    add(t.y0, t.x0, t.w00);
    add(t.y0, t.x1, t.w01);
    add(t.y1, t.x0, t.w10);
    add(t.y1, t.x1, t.w11);
    ifu_st8(out + pix * 64 + v * 8, acc);
  }
}

// the frame: r_b = clamp(rwarp_b + tanh(decode_b), 0, 1) (decode: ConvT phases ph [4][2][h][w][4], grid 2h x 2w = Hp x
// Wp); p = softmax(clamp(m0), clamp(m1), 0) over [-4, 4]; out = r0 p0 + r1 p1 + deg p2 on the H x W crop
__global__ void ifu_final_kernel(const float* __restrict__ ph, const float* __restrict__ rwarp,
                                 const float* __restrict__ rmask, const float* __restrict__ deg, int H, int W, int Hp,
                                 int Wp, float* __restrict__ out) {
  const size_t plane = (size_t)Hp * Wp, total = (size_t)H * W;
  const int h = Hp / 2, w = Wp / 2;
  const size_t pl = (size_t)2 * h * w * 4;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W), y = (int)(i / W);
    const size_t p = (size_t)y * Wp + x;
    const int q = (y & 1) * 2 + (x & 1);
    float m[3];
    for (int b = 0; b < 2; ++b) m[b] = fminf(fmaxf(rmask[b * plane + p], -4.f), 4.f);
    m[2] = 0.f;
    const float mx = fmaxf(fmaxf(m[0], m[1]), m[2]);
    float e[3], den = 0.f;
    for (int k = 0; k < 3; ++k) {
      e[k] = expf(m[k] - mx);
      den += e[k];
    }
    for (int c = 0; c < 3; ++c) {
      float acc = 0.f;
      for (int b = 0; b < 2; ++b) {
        const float d = ph[q * pl + (((size_t)b * h + (y >> 1)) * w + (x >> 1)) * 4 + c];
        const float r = fminf(fmaxf(rwarp[(b * 3 + c) * plane + p] + tanhf(d), 0.f), 1.f);
        acc += r * (e[b] / den);
      }
      acc += deg[c * plane + p] * (e[2] / den);
      out[(size_t)c * H * W + i] = acc;
    }
  }
}

}  // namespace


cudaError_t launch_ifunet_flow_in(int op, const IfuFlowIn& a, int B, void* out, cudaStream_t st) {
  const int g = ifu_grid((size_t)B * ((a.h0 + 1) / 2) * ((a.w0 + 1) / 2) * 4, 128);
  if (op == OP_BF16)
    VFI_LAUNCH(ifu_flow_in_kernel<__nv_bfloat16>, g, 128, 0, st, a, B, (__nv_bfloat16*)out);
  else
    VFI_LAUNCH(ifu_flow_in_kernel<__half>, g, 128, 0, st, a, B, (__half*)out);
  return cudaGetLastError();
}

cudaError_t launch_ifunet_s2d(int op, const void* in, int pitch, int cq, int B, int h, int w, void* out, int opitch,
                              cudaStream_t st) {
  const int g = ifu_grid((size_t)B * ((h + 1) / 2) * ((w + 1) / 2) * (opitch / 8), 256);
  if (op == OP_BF16)
    VFI_LAUNCH(ifu_s2d_kernel<__nv_bfloat16>, g, 256, 0, st, (const __nv_bfloat16*)in, pitch, cq, B, h, w,
               (__nv_bfloat16*)out, opitch);
  else
    VFI_LAUNCH(ifu_s2d_kernel<__half>, g, 256, 0, st, (const __half*)in, pitch, cq, B, h, w, (__half*)out, opitch);
  return cudaGetLastError();
}

cudaError_t launch_ifunet_d2s(const void* ph, int C, int B, int h, int w, void* out, cudaStream_t st) {
  if (C & 7) return cudaErrorInvalidValue;
  VFI_LAUNCH(ifu_d2s_kernel, ifu_grid((size_t)B * 4 * h * w * (C / 8), 256), 256, 0, st, (const uint4*)ph, C / 8, B, h, w,
             (uint4*)out);
  return cudaGetLastError();
}

cudaError_t launch_ifunet_cbam(int op, void* x, int pitch, int C, int B, int h, int w, const float* mlp, const float* sw,
                               float* psum, float* pmax, float* gate, float* cmp, cudaStream_t st) {
  if ((C & 7) || C > 512 || C < 16) return cudaErrorInvalidValue;
  const int npx = h * w, threads = 256;
  const dim3 pg(kIfuPoolChunks, B);
  const int g = ifu_grid((size_t)B * npx, 256), g2 = ifu_grid((size_t)B * npx * (C / 8), 256);
  if (op == OP_BF16) {
    VFI_LAUNCH(ifu_pool_kernel<__nv_bfloat16>, pg, threads, 0, st, (const __nv_bfloat16*)x, pitch, C, npx, psum, pmax);
    VFI_LAUNCH(ifu_gate_kernel, B, 256, 0, st, psum, pmax, C, C / 16, npx, B, mlp, gate);
    VFI_LAUNCH(ifu_compress_kernel<__nv_bfloat16>, g, 256, 0, st, (const __nv_bfloat16*)x, pitch, C, B, npx, gate,
               (float2*)cmp);
    VFI_LAUNCH(ifu_spatial_kernel<__nv_bfloat16>, g2, 256, 0, st, (const __nv_bfloat16*)x, pitch, C, B, h, w, gate,
               (const float2*)cmp, sw, (__nv_bfloat16*)x);
  } else {
    VFI_LAUNCH(ifu_pool_kernel<__half>, pg, threads, 0, st, (const __half*)x, pitch, C, npx, psum, pmax);
    VFI_LAUNCH(ifu_gate_kernel, B, 256, 0, st, psum, pmax, C, C / 16, npx, B, mlp, gate);
    VFI_LAUNCH(ifu_compress_kernel<__half>, g, 256, 0, st, (const __half*)x, pitch, C, B, npx, gate, (float2*)cmp);
    VFI_LAUNCH(ifu_spatial_kernel<__half>, g2, 256, 0, st, (const __half*)x, pitch, C, B, h, w, gate, (const float2*)cmp, sw,
               (__half*)x);
  }
  return cudaGetLastError();
}

cudaError_t launch_ifunet_add16(int op, void* x, const void* y, size_t n, cudaStream_t st) {
  if (n & 7) return cudaErrorInvalidValue;
  const int g = ifu_grid(n / 8, 256);
  if (op == OP_BF16)
    VFI_LAUNCH(ifu_add_kernel<__nv_bfloat16>, g, 256, 0, st, (__nv_bfloat16*)x, (const __nv_bfloat16*)y, n / 8);
  else
    VFI_LAUNCH(ifu_add_kernel<__half>, g, 256, 0, st, (__half*)x, (const __half*)y, n / 8);
  return cudaGetLastError();
}

cudaError_t launch_ifunet_convex(int op, const float* flow, const void* mask, int L, int B, int h, int w, float* up,
                                 cudaStream_t st) {
  const int g = ifu_grid((size_t)B * L * h * L * w, 256);
  if (op == OP_BF16)
    VFI_LAUNCH(ifu_convex_kernel<__nv_bfloat16>, g, 256, 0, st, flow, (const __nv_bfloat16*)mask, L, B, h, w, up);
  else
    VFI_LAUNCH(ifu_convex_kernel<__half>, g, 256, 0, st, flow, (const __half*)mask, L, B, h, w, up);
  return cudaGetLastError();
}

cudaError_t launch_ifunet_flow_update(const float* up, int uh, int uw, int resize, float cscale, float fmul, int mode,
                                      int Hp, int Wp, float* flow, cudaStream_t st) {
  if (mode < 0 || mode > 3) return cudaErrorInvalidValue;
  VFI_LAUNCH(ifu_flow_update_kernel, ifu_grid((size_t)Hp * Wp, 256), 256, 0, st, (const float4*)up, uh, uw, resize, cscale,
             fmul, mode, Hp, Wp, (float4*)flow);
  return cudaGetLastError();
}

cudaError_t launch_ifunet_warp_frames(const float* f0, const float* f1, int H, int W, int Hp, int Wp, const float* flow,
                                      float* warped, cudaStream_t st) {
  VFI_LAUNCH(ifu_warp_frames_kernel, ifu_grid((size_t)Hp * Wp, 256), 256, 0, st, f0, f1, H, W, Hp, Wp,
             (const float4*)flow, warped);
  return cudaGetLastError();
}

cudaError_t launch_ifunet_fusion_in(int op, const float* f0, const float* f1, int H, int W, int Hp, int Wp,
                                    const float* warped, const float* flow, void* out, cudaStream_t st) {
  const int g = ifu_grid((size_t)(Hp / 4) * (Wp / 4), 128);
  if (op == OP_BF16)
    VFI_LAUNCH(ifu_fusion_in_kernel<__nv_bfloat16>, g, 128, 0, st, f0, f1, H, W, Hp, Wp, warped, (const float4*)flow,
               (__nv_bfloat16*)out);
  else
    VFI_LAUNCH(ifu_fusion_in_kernel<__half>, g, 128, 0, st, f0, f1, H, W, Hp, Wp, warped, (const float4*)flow,
               (__half*)out);
  return cudaGetLastError();
}

cudaError_t launch_ifunet_rrdb_res(int op, void* y, const void* x, size_t n, cudaStream_t st) {
  if (n & 7) return cudaErrorInvalidValue;
  const int g = ifu_grid(n / 8, 256);
  if (op == OP_BF16)
    VFI_LAUNCH(ifu_rrdb_res_kernel<__nv_bfloat16>, g, 256, 0, st, (__nv_bfloat16*)y, (const __nv_bfloat16*)x, n / 8);
  else
    VFI_LAUNCH(ifu_rrdb_res_kernel<__half>, g, 256, 0, st, (__half*)y, (const __half*)x, n / 8);
  return cudaGetLastError();
}

cudaError_t launch_ifunet_merge(const float* warped, const float* last, int Hp, int Wp, float* deg, cudaStream_t st) {
  VFI_LAUNCH(ifu_merge_kernel, ifu_grid((size_t)Hp * Wp, 256), 256, 0, st, warped, last, Hp, Wp, deg);
  return cudaGetLastError();
}

cudaError_t launch_ifunet_fb_in(const float* f0, const float* f1, int H, int W, int Hp, int Wp, const float* deg,
                                const float* rwarp, const float* rmask, const float* rflow, int cin, int s, float* out,
                                cudaStream_t st) {
  if (cin != 6 && cin != 12) return cudaErrorInvalidValue;
  VFI_LAUNCH(ifu_fb_in_kernel, ifu_grid((size_t)2 * (Hp / s) * (Wp / s), 256), 256, 0, st, f0, f1, H, W, Hp, Wp, deg, rwarp,
             rmask, (const float2*)rflow, cin, s, out);
  return cudaGetLastError();
}

cudaError_t launch_ifunet_stem(int op, const float* src0, const float* src1, int cin, int sh, int sw, int vh, int vw,
                               const float* w, const float* bias, const float* slopes, int cout, int B, int pitch, void* out,
                               cudaStream_t st) {
  if ((pitch & 7) || cout > pitch) return cudaErrorInvalidValue;
  const int ho = (sh + 1) / 2, wo = (sw + 1) / 2;
  StemSrc s{{src0, src1}};
  const int g = ifu_grid((size_t)B * ho * wo * (pitch / 8), 128);
  if (op == OP_BF16)
    VFI_LAUNCH(ifu_stem_kernel<__nv_bfloat16>, g, 128, 0, st, s, cin, sh, sw, vh, vw, w, bias, slopes, cout, B, ho, wo, pitch,
               (__nv_bfloat16*)out);
  else
    VFI_LAUNCH(ifu_stem_kernel<__half>, g, 128, 0, st, s, cin, sh, sw, vh, vw, w, bias, slopes, cout, B, ho, wo, pitch,
               (__half*)out);
  return cudaGetLastError();
}

cudaError_t launch_ifunet_fb_out(const float* ph, int h, int w, int s, int first, const float* f0, const float* f1, int H,
                                 int W, int Hp, int Wp, float* rflow, float* rmask, float* rwarp, cudaStream_t st) {
  VFI_LAUNCH(ifu_fb_out_kernel, ifu_grid((size_t)2 * Hp * Wp, 256), 256, 0, st, ph, h, w, s, first, f0, f1, H, W, Hp, Wp,
             (float2*)rflow, rmask, rwarp);
  return cudaGetLastError();
}

cudaError_t launch_ifunet_ctx_warp(int op, const void* feat, int fpitch, const float* rflow, int Hp, int Wp, void* out,
                                   cudaStream_t st) {
  const int g = ifu_grid((size_t)2 * (Hp / 4) * (Wp / 4) * 4, 256);
  if (op == OP_BF16)
    VFI_LAUNCH(ifu_ctx_warp_kernel<__nv_bfloat16>, g, 256, 0, st, (const __nv_bfloat16*)feat, fpitch, (const float2*)rflow,
               Hp, Wp, (__nv_bfloat16*)out);
  else
    VFI_LAUNCH(ifu_ctx_warp_kernel<__half>, g, 256, 0, st, (const __half*)feat, fpitch, (const float2*)rflow, Hp, Wp,
               (__half*)out);
  return cudaGetLastError();
}

cudaError_t launch_ifunet_final(const float* ph, const float* rwarp, const float* rmask, const float* deg, int H, int W,
                                int Hp, int Wp, float* out, cudaStream_t st) {
  VFI_LAUNCH(ifu_final_kernel, ifu_grid((size_t)H * W, 256), 256, 0, st, ph, rwarp, rmask, deg, H, W, Hp, Wp, out);
  return cudaGetLastError();
}

}  // namespace vfi
