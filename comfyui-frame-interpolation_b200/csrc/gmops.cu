// gmops: the fp32 building blocks of the GMFSS Fortuna path (SURVEY.md section 8 row a11), CUDA cores, NCHW like the
// reference's tensors.  Everything GMFSS_Fortuna_union_arch.py does with ATen / cuDNN / cuBLAS between its custom
// softsplat calls is one of these kernels (the schedule itself is host code: comfyui-frame-interpolation_b200/gmfss.py):
//   conv2d / conv_transpose2d(4, 2, 1) with the PReLU that precedes them and the residual adds that follow them fused
//     (MetricNet :1420-1467, FeatureNet :1470-1500, GridNet :1503-1688, GMFlow's CNNEncoder :165-312, upsampler :1190-1199)
//   instance_norm (+ReLU), add+ReLU                                   (ResidualBlock_class :165-215)
//   gemm (q / k / v / merge / MLP linears, attention scores and products), row softmax, layer_norm + residual
//     (TransformerLayer :439-523, FeatureFlowAttention :688-803, global_correlation_softmax :806-843)
//   window split / merge with the cyclic shift                         (split_feature / merge_splits :1059-1131, :366-436)
//   sine position embedding                                            (PositionEmbeddingSine :1015-1056)
//   local correlation softmax (radius 4) and local flow propagation (radius 1)       (:846-913, :757-803)
//   convex up-sampling                                                 (GMFlow.upsample_flow :1220-1260)
//   bilinear resampling: warp with zero padding (flow_warp :955-991, backwarp :1375-1417), resize (F.interpolate)
//   MetricNet's 14-channel input (photometric errors, normalised flows, forward-backward occlusion; :1429-1455, :994-1013)
//   pixel shuffle, scaled adds.
// First version: correct and simple - one thread per small output tile with register blocking, operands through L1 (no
// shared-memory staging, no tensor cores); its parity is pinned on the CPU through tests/host_emu before any GPU run.
#include <cmath>
#include <cstdint>
#include <string>

#include "../../include/vfi_b200.h"
#include "vfi_internal.h"

namespace vfi {
namespace {

constexpr int kThreads = 128;

inline int grid_for_n(size_t total, int block) {
  size_t g = (total + block - 1) / block;
  if (g < 1) g = 1;
  if (g > 65535u * 16u) g = 65535u * 16u;
  return (int)g;
}

__device__ __forceinline__ float act_pre(float v, int has, float slope) { return (has && v < 0.f) ? v * slope : v; }

// ------------------------------------------------------------------------------------------------ conv2d
// out[n, out_coff + co, yo, xo] = post( bias[co] + sum_{ci,ky,kx} pre(in[n, in_coff + ci, yo*s - pad + ky, xo*s - pad + kx]) * w[co, ci, ky, kx]
//                                       + res1 + res2 )
// thread = (n, 16 output channels, yo, 4 consecutive xo)
__global__ void conv2d_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                              const float* __restrict__ res1, const float* __restrict__ res2, float* __restrict__ out, int N,
                              int Cin, int H, int W, int Cout, int Ho, int Wo, int k, int stride, int pad, int in_ctot, int in_coff,
                              int out_ctot, int out_coff, int has_pre, float pre_slope, int post, float post_slope) {
  const int cog = (Cout + 15) / 16, xq = (Wo + 3) / 4;
  const size_t total = (size_t)N * cog * Ho * xq;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int xo0 = (int)(id % xq) * 4;
    size_t r = id / xq;
    const int yo = (int)(r % Ho);
    r /= Ho;
    const int co0 = (int)(r % cog) * 16;
    const int n = (int)(r / cog);
    float acc[4][16];
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[p][j] = 0.f;
    const size_t wstride = (size_t)Cin * k * k;
    for (int ci = 0; ci < Cin; ++ci) {
      const float* ip = in + ((size_t)n * in_ctot + in_coff + ci) * H * W;
      for (int ky = 0; ky < k; ++ky) {
        const int yi = yo * stride - pad + ky;
        if (yi < 0 || yi >= H) continue;
        for (int kx = 0; kx < k; ++kx) {
          float v[4];
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            const int xi = (xo0 + p) * stride - pad + kx;
            v[p] = (xi >= 0 && xi < W && xo0 + p < Wo) ? act_pre(__ldg(ip + (size_t)yi * W + xi), has_pre, pre_slope) : 0.f;
          }
          const float* wp = w + ((size_t)co0 * Cin + ci) * k * k + ky * k + kx;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const float wj = (co0 + j < Cout) ? __ldg(wp + (size_t)j * wstride) : 0.f;
#pragma unroll
            for (int p = 0; p < 4; ++p) acc[p][j] = fmaf(v[p], wj, acc[p][j]);
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int co = co0 + j;
      if (co >= Cout) break;
      const float b = bias ? __ldg(bias + co) : 0.f;
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const int xo = xo0 + p;
        if (xo >= Wo) continue;
        float v = acc[p][j] + b;
        const size_t ro = (((size_t)n * Cout + co) * Ho + yo) * Wo + xo;
        if (res1) v += res1[ro];
        if (res2) v += res2[ro];
        if (post == 1) v = fmaxf(v, 0.f);
        else if (post == 2) v = tanhf(v) * 10.f;
        else if (post == 3) v = v < 0.f ? v * post_slope : v;
        out[(((size_t)n * out_ctot + out_coff + co) * Ho + yo) * Wo + xo] = v;
      }
    }
  }
}

// The same convolution, the form the heavy layers run in: weights re-packed once at load time to wt[(ci, ky, kx)][CoutP]
// (output channel fastest, padded to a multiple of 16, gmfss.Ops.pack_conv) so that the 16 weights of a tap are four 16-byte
// loads; thread = (n, 16 output channels, yo, PX = 8 consecutive xo); per (ci, ky) the input row segment the 8 pixels need
// is loaded once into registers and reused by all kx taps: (7 S + K) + 4 K loads for 128 K multiply-adds, K and the stride S
// compile-time so that everything stays in registers (the scalar-weight form above loads one weight per four multiply-adds).
template <int K, int S>
__global__ void conv2d_packed_kernel(const float* __restrict__ in, const float* __restrict__ wt, const float* __restrict__ bias,
                                     const float* __restrict__ res1, const float* __restrict__ res2, float* __restrict__ out, int N,
                                     int Cin, int H, int W, int Cout, int CoutP, int Ho, int Wo, int pad, int in_ctot, int in_coff,
                                     int out_ctot, int out_coff, int has_pre, float pre_slope, int post, float post_slope) {
  constexpr int PX = 8, SEG = (PX - 1) * S + K;
  const int cog = CoutP / 16, xq = (Wo + PX - 1) / PX;
  const size_t total = (size_t)N * cog * Ho * xq;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int xo0 = (int)(id % xq) * PX;
    size_t r = id / xq;
    const int yo = (int)(r % Ho);
    r /= Ho;
    const int co0 = (int)(r % cog) * 16;
    const int n = (int)(r / cog);
    float acc[PX][16];
#pragma unroll
    for (int p = 0; p < PX; ++p)
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[p][j] = 0.f;
    const int xs = xo0 * S - pad;
    for (int ci = 0; ci < Cin; ++ci) {
      const float* ip = in + ((size_t)n * in_ctot + in_coff + ci) * H * W;
#pragma unroll
      for (int ky = 0; ky < K; ++ky) {
        const int yi = yo * S - pad + ky;
        if (yi < 0 || yi >= H) continue;
        float seg[SEG];
#pragma unroll
        for (int i = 0; i < SEG; ++i) {
          const int xi = xs + i;
          seg[i] = (xi >= 0 && xi < W) ? act_pre(__ldg(ip + (size_t)yi * W + xi), has_pre, pre_slope) : 0.f;
        }
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
          const float4* wp = reinterpret_cast<const float4*>(wt + ((size_t)(ci * K + ky) * K + kx) * CoutP + co0);
          const float4 w0 = __ldg(wp), w1 = __ldg(wp + 1), w2 = __ldg(wp + 2), w3 = __ldg(wp + 3);
          const float wv[16] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w, w2.x, w2.y, w2.z, w2.w, w3.x, w3.y, w3.z, w3.w};
#pragma unroll
          for (int p = 0; p < PX; ++p) {
            const float v = seg[p * S + kx];
#pragma unroll
            for (int j = 0; j < 16; ++j) acc[p][j] = fmaf(v, wv[j], acc[p][j]);
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int co = co0 + j;
      if (co < Cout) {
        const float b = bias ? __ldg(bias + co) : 0.f;
#pragma unroll
        for (int p = 0; p < PX; ++p) {
          const int xo = xo0 + p;
          if (xo < Wo) {
            float v = acc[p][j] + b;
            const size_t ro = (((size_t)n * Cout + co) * Ho + yo) * Wo + xo;
            if (res1) v += res1[ro];
            if (res2) v += res2[ro];
            if (post == 1) v = fmaxf(v, 0.f);
            else if (post == 2) v = tanhf(v) * 10.f;
            else if (post == 3) v = v < 0.f ? v * post_slope : v;
            out[(((size_t)n * out_ctot + out_coff + co) * Ho + yo) * Wo + xo] = v;
          }
        }
      }
    }
  }
}

// ConvTranspose2d(Cin, Cout, 4, stride 2, padding 1) with the preceding PReLU: w [Cin, Cout, 4, 4], out [N, Cout, 2H, 2W]:
// out[yo, xo] += in[yi, xi] * w[ky, kx] with yo = 2 yi - 1 + ky.  thread = (n, 16 output channels, yo, 4 consecutive xo)
__global__ void convt4_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                              float* __restrict__ out, int N, int Cin, int H, int W, int Cout, int has_pre, float pre_slope) {
  const int Ho = 2 * H, Wo = 2 * W;
  const int cog = (Cout + 15) / 16, xq = (Wo + 3) / 4;
  const size_t total = (size_t)N * cog * Ho * xq;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int xo0 = (int)(id % xq) * 4;
    size_t r = id / xq;
    const int yo = (int)(r % Ho);
    r /= Ho;
    const int co0 = (int)(r % cog) * 16;
    const int n = (int)(r / cog);
    float acc[4][16];
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[p][j] = 0.f;
    for (int ci = 0; ci < Cin; ++ci) {
      const float* ip = in + ((size_t)n * Cin + ci) * H * W;
      const float* wc = w + ((size_t)ci * Cout + co0) * 16;
      for (int ky = (yo + 1) & 1; ky < 4; ky += 2) {
        const int yi = (yo + 1 - ky) >> 1;  // exact: yo + 1 - ky is even
        if (yo + 1 - ky < 0 || yi >= H) continue;
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const int xo = xo0 + p;
          if (xo >= Wo) continue;
          for (int kx = (xo + 1) & 1; kx < 4; kx += 2) {
            const int xi = (xo + 1 - kx) >> 1;
            if (xo + 1 - kx < 0 || xi >= W) continue;
            const float v = act_pre(__ldg(ip + (size_t)yi * W + xi), has_pre, pre_slope);
#pragma unroll
            for (int j = 0; j < 16; ++j)
              if (co0 + j < Cout) acc[p][j] = fmaf(v, __ldg(wc + j * 16 + ky * 4 + kx), acc[p][j]);
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int co = co0 + j;
      if (co >= Cout) break;
      const float b = bias ? __ldg(bias + co) : 0.f;
#pragma unroll
      for (int p = 0; p < 4; ++p)
        if (xo0 + p < Wo) out[(((size_t)n * Cout + co) * Ho + yo) * Wo + xo0 + p] = acc[p][j] + b;
    }
  }
}

// ------------------------------------------------------------------------------------------------ normalisations
// InstanceNorm2d(affine=False, eps): one block per (n, c) plane; optional ReLU
__global__ void instance_norm_kernel(const float* __restrict__ in, float* __restrict__ out, int HW, float eps, int relu) {
  __shared__ float red[kThreads];
  const float* p = in + (size_t)blockIdx.x * HW;
  float* q = out + (size_t)blockIdx.x * HW;
  float s = 0.f;
  for (int i = threadIdx.x; i < HW; i += blockDim.x) s += p[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  const float mean = red[0] / (float)HW;
  __syncthreads();
  float v = 0.f;
  for (int i = threadIdx.x; i < HW; i += blockDim.x) {
    const float d = p[i] - mean;
    v += d * d;
  }
  red[threadIdx.x] = v;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  const float rstd = (1.f / sqrtf(red[0] / (float)HW + eps));
  for (int i = threadIdx.x; i < HW; i += blockDim.x) {
    float y = (p[i] - mean) * rstd;
    if (relu) y = fmaxf(y, 0.f);
    q[i] = y;
  }
}

// out = src + LayerNorm(x) over the last dimension C (one block per row; src may be null: out = LN(x))
__global__ void layer_norm_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                                  const float* __restrict__ src, float* __restrict__ out, int C, float eps) {
  __shared__ float red[kThreads];
  const float* p = x + (size_t)blockIdx.x * C;
  float s = 0.f;
  for (int i = threadIdx.x; i < C; i += blockDim.x) s += p[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  const float mean = red[0] / (float)C;
  __syncthreads();
  float v = 0.f;
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    const float d = p[i] - mean;
    v += d * d;
  }
  red[threadIdx.x] = v;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  const float rstd = (1.f / sqrtf(red[0] / (float)C + eps));
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    const float y = (p[i] - mean) * rstd * gamma[i] + beta[i];
    out[(size_t)blockIdx.x * C + i] = (src ? src[(size_t)blockIdx.x * C + i] : 0.f) + y;
  }
}

// row softmax in place: one block per row of length L
__global__ void softmax_rows_kernel(float* __restrict__ x, int L) {
  __shared__ float red[kThreads];
  float* p = x + (size_t)blockIdx.x * L;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < L; i += blockDim.x) m = fmaxf(m, p[i]);
  red[threadIdx.x] = m;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + o]);
    __syncthreads();
  }
  m = red[0];
  __syncthreads();
  float s = 0.f;
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    const float e = expf(p[i] - m);
    p[i] = e;
    s += e;
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  const float inv = 1.f / red[0];
  for (int i = threadIdx.x; i < L; i += blockDim.x) p[i] *= inv;
}

// ------------------------------------------------------------------------------------------------ gemm
// C[b][m][n] = act( alpha * sum_k A[b][m][k] * (BT ? B[b][n][k] : B[b][k][n]) + bias[n] + mask[b % nmask][m][n] )
// thread = (b, 8 rows, 2 columns n and n + 32 * ...): lanes run along n
template <bool BT>
__global__ void gemm_kernel(const float* __restrict__ A, const float* __restrict__ B, const float* __restrict__ bias,
                            const float* __restrict__ mask, float* __restrict__ C, int nb, int M, int N, int K, int lda, int ldb,
                            int ldc, long long sA, long long sB, long long sC, float alpha, int nmask, int act) {
  const int mq = (M + 7) / 8;
  const size_t total = (size_t)nb * mq * N;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(id % N);
    size_t r = id / N;
    const int m0 = (int)(r % mq) * 8;
    const int b = (int)(r / mq);
    const float* a = A + (size_t)b * sA + (size_t)m0 * lda;
    const float* bp = B + (size_t)b * sB;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    const int rows = min(8, M - m0);
    for (int k = 0; k < K; ++k) {
      const float bv = BT ? __ldg(bp + (size_t)n * ldb + k) : __ldg(bp + (size_t)k * ldb + n);
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (i < rows) acc[i] = fmaf(__ldg(a + (size_t)i * lda + k), bv, acc[i]);
    }
    const float bs = bias ? __ldg(bias + n) : 0.f;
    for (int i = 0; i < rows; ++i) {
      float v = acc[i] * alpha + bs;
      if (mask) v += __ldg(mask + ((size_t)(b % nmask) * M + m0 + i) * N + n);
      if (act == 1) v = 0.5f * v * (1.f + erff(v * 0.70710678118654752f));  // GELU (erf form, nn.GELU default)
      C[(size_t)b * sC + (size_t)(m0 + i) * ldc + n] = v;
    }
  }
}

// C[b][m][n] = act( alpha * sum_k A[b][m][k] * B[b][k][n] + bias[n] + mask[b % nmask][m][n] ), the form the heavy products run
// in (linears with the weight transposed once at load time, attention scores against the transposed keys, P V): thread = an
// 8 x 8 tile of C, lanes along n; per four k: eight 16-byte loads of A (one per row, the same for every lane of a row group)
// and eight of B (coalesced) for 256 multiply-adds.  Needs K % 4 == 0, N % 8 == 0, 16-byte aligned rows.
template <int MT>
__global__ void gemm_nn8_kernel(const float* __restrict__ A, const float* __restrict__ B, const float* __restrict__ bias,
                                const float* __restrict__ mask, float* __restrict__ C, int nb, int M, int N, int K, int lda, int ldb,
                                int ldc, long long sA, long long sB, long long sC, float alpha, int nmask, int act) {
  const int mq = (M + MT - 1) / MT, nq = N / 8;
  const size_t total = (size_t)nb * mq * nq;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int n0 = (int)(id % nq) * 8;
    size_t r = id / nq;
    const int m0 = (int)(r % mq) * MT;
    const int b = (int)(r / mq);
    const float* a = A + (size_t)b * sA;
    const float* bp = B + (size_t)b * sB + n0;
    float acc[MT][8];
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    int row[MT];
#pragma unroll
    for (int i = 0; i < MT; ++i) row[i] = min(m0 + i, M - 1);  // rows past M recompute the last one and are not stored
    for (int k = 0; k < K; k += 4) {
      float4 av[MT];
#pragma unroll
      for (int i = 0; i < MT; ++i) av[i] = __ldg(reinterpret_cast<const float4*>(a + (size_t)row[i] * lda + k));
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(bp + (size_t)(k + kk) * ldb));
        const float4 b1 = __ldg(reinterpret_cast<const float4*>(bp + (size_t)(k + kk) * ldb + 4));
        const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int i = 0; i < MT; ++i) {
          const float x = kk == 0 ? av[i].x : kk == 1 ? av[i].y : kk == 2 ? av[i].z : av[i].w;
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(x, bv[j], acc[i][j]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < MT; ++i) {
      if (m0 + i < M) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float v = acc[i][j] * alpha + (bias ? __ldg(bias + n0 + j) : 0.f);
          if (mask) v += __ldg(mask + ((size_t)(b % nmask) * M + m0 + i) * N + n0 + j);
          if (act == 1) v = 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
          C[(size_t)b * sC + (size_t)(m0 + i) * ldc + n0 + j] = v;
        }
      }
    }
  }
}

// [nb, R, C] -> [nb, C, R]
__global__ void transpose_kernel(const float* __restrict__ src, float* __restrict__ dst, int nb, int R, int C) {
  const size_t total = (size_t)nb * R * C;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int rr = (int)(id % R);
    size_t q = id / R;
    const int c = (int)(q % C);
    const int b = (int)(q / C);
    dst[id] = src[((size_t)b * R + rr) * C + c];
  }
}

// ------------------------------------------------------------------------------------------------ token <-> window layout
// tokens [B, H, W, C] (row-major over h, w)  <->  windows [B * k * k, (H/k) * (W/k), C]; with a cyclic shift (sh, sw):
// forward: win[...] = tok[(y + sh) mod H, (x + sw) mod W]  (torch.roll by (-sh, -sw) then split); backward undoes both
__global__ void window_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int H, int W, int C, int k, int sh,
                              int sw, int to_windows) {
  const int hh = H / k, ww = W / k;
  const size_t total = (size_t)B * H * W * C;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(id % C);
    size_t r = id / C;
    const int x = (int)(r % W);
    r /= W;
    const int y = (int)(r % H);
    const int b = (int)(r / H);
    // (y, x) = position in the SHIFTED image; its window and the source position in the unshifted token grid
    const int wy = y / hh, wx = x / ww, iy = y - wy * hh, ix = x - wx * ww;
    const size_t widx = ((((size_t)b * k + wy) * k + wx) * (size_t)(hh * ww) + (size_t)iy * ww + ix) * C + c;
    const int ys = (y + sh) % H, xs = (x + sw) % W;
    const size_t tidx = (((size_t)b * H + ys) * W + xs) * C + c;
    if (to_windows) dst[widx] = src[tidx];
    else dst[tidx] = src[widx];
  }
}

// NCHW [B, C, H, W] <-> tokens [B, H*W, C]
__global__ void nchw_tokens_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int C, int HW, int to_tokens) {
  const size_t total = (size_t)B * C * HW;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int p = (int)(id % HW);
    size_t r = id / HW;
    const int c = (int)(r % C);
    const int b = (int)(r / C);
    const size_t t = ((size_t)b * HW + p) * C + c;
    if (to_tokens) dst[t] = src[id];
    else dst[id] = src[t];
  }
}

// x[b, c, y, x] += PositionEmbeddingSine(C/2 feats, temperature 10000, normalize) evaluated per WINDOW of (H/k) x (W/k)
// (feature_add_position :1134-1154 splits, adds, merges): channels [0, C/2) from y, [C/2, C) from x
__global__ void add_position_kernel(float* __restrict__ x, int B, int C, int H, int W, int k) {
  const int hh = H / k, ww = W / k, F = C / 2;
  const size_t total = (size_t)B * C * H * W;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int xx = (int)(id % W);
    size_t r = id / W;
    const int yy = (int)(r % H);
    r /= H;
    const int c = (int)(r % C);
    const int iy = yy % hh, ix = xx % ww;
    const bool isy = c < F;
    const int f = isy ? c : c - F;
    const float e = isy ? (float)(iy + 1) / ((float)hh + 1e-6f) : (float)(ix + 1) / ((float)ww + 1e-6f);
    const float dim_t = powf(10000.f, (float)(2 * (f / 2)) / (float)F);
    const float arg = e * 6.283185307179586f / dim_t;
    x[id] += (f & 1) ? cosf(arg) : sinf(arg);
  }
}

// ------------------------------------------------------------------------------------------------ matching
// local_correlation_softmax :846-913 with radius R: flow[b, :, y, x] = sum_d softmax_d( <f0(y,x), f1(y+dy, x+dx)> / sqrt(C) ) * (dx, dy)
// (out-of-image displacements get -1e9 before the softmax; the sampled feature there is zero).  feats NCHW.
__global__ void local_match_kernel(const float* __restrict__ f0, const float* __restrict__ f1, float* __restrict__ flow, int B, int C,
                                   int H, int W, int R) {
  const int K = 2 * R + 1;
  const size_t total = (size_t)B * H * W;
  const float scale = (1.f / sqrtf((float)C));
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(id % W);
    size_t r = id / W;
    const int y = (int)(r % H);
    const int b = (int)(r / H);
    const float* a = f0 + (size_t)b * C * H * W + (size_t)y * W + x;
    const float* g = f1 + (size_t)b * C * H * W;
    float mx = -INFINITY;
    float corr[81];
    for (int d = 0; d < K * K; ++d) {
      const int dy = d / K - R, dx = d % K - R;   // window order: the reference's (x fastest) grid, :870-876
      const int yy = y + dy, xx = x + dx;
      float s = -1e9f;
      if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
        s = 0.f;
        for (int c = 0; c < C; ++c) s = fmaf(a[(size_t)c * H * W], g[(size_t)c * H * W + (size_t)yy * W + xx], s);
        s *= scale;
      }
      corr[d] = s;
      mx = fmaxf(mx, s);
    }
    float den = 0.f, fx = 0.f, fy = 0.f;
    for (int d = 0; d < K * K; ++d) {
      const float e = expf(corr[d] - mx);
      den += e;
      fx += e * (float)(x + d % K - R);
      fy += e * (float)(y + d / K - R);
    }
    flow[((size_t)b * 2 + 0) * H * W + (size_t)y * W + x] = fx / den - (float)x;
    flow[((size_t)b * 2 + 1) * H * W + (size_t)y * W + x] = fy / den - (float)y;
  }
}

// FeatureFlowAttention.forward_local_window_attn :757-803, radius 1: q, k tokens [B, H*W, C] (already projected), flow NCHW;
// out[b, :, y, x] = sum_{3x3} softmax( <q(y,x), k(y+dy,x+dx)> / sqrt(C) ) * flow(y+dy, x+dx), zero padding for k and flow
__global__ void local_prop_kernel(const float* __restrict__ q, const float* __restrict__ kk, const float* __restrict__ flow,
                                  float* __restrict__ out, int B, int C, int H, int W) {
  const size_t total = (size_t)B * H * W;
  const float scale = (1.f / sqrtf((float)C));
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(id % W);
    size_t r = id / W;
    const int y = (int)(r % H);
    const int b = (int)(r / H);
    const float* qp = q + id * C;
    float s[9], mx = -INFINITY;
    for (int d = 0; d < 9; ++d) {
      const int yy = y + d / 3 - 1, xx = x + d % 3 - 1;
      float v = 0.f;  // F.unfold pads the key map with zeros: the score of an outside tap is 0, not -inf
      if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
        const float* kp = kk + (((size_t)b * H + yy) * W + xx) * C;
        for (int c = 0; c < C; ++c) v = fmaf(qp[c], kp[c], v);
      }
      s[d] = v * scale;
      mx = fmaxf(mx, s[d]);
    }
    float den = 0.f, fx = 0.f, fy = 0.f;
    for (int d = 0; d < 9; ++d) {
      const int yy = y + d / 3 - 1, xx = x + d % 3 - 1;
      const float e = expf(s[d] - mx);
      den += e;
      if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
        fx += e * flow[((size_t)b * 2 + 0) * H * W + (size_t)yy * W + xx];
        fy += e * flow[((size_t)b * 2 + 1) * H * W + (size_t)yy * W + xx];
      }
    }
    out[((size_t)b * 2 + 0) * H * W + (size_t)y * W + x] = fx / den;
    out[((size_t)b * 2 + 1) * H * W + (size_t)y * W + x] = fy / den;
  }
}

// GMFlow.upsample_flow :1220-1260: mask [B, 9 * f * f, H, W] (raw conv output), flow [B, 2, H, W] -> up [B, 2, f H, f W]:
// softmax over the 9 taps of channel (t, fy, fx), up[y f + fy, x f + fx] = sum_t p_t * f * flow(3x3 neighbour t, zero padded)
__global__ void convex_up_kernel(const float* __restrict__ mask, const float* __restrict__ flow, float* __restrict__ up, int B, int H,
                                 int W, int f) {
  const size_t total = (size_t)B * H * W * f * f;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int fx = (int)(id % f);
    size_t r = id / f;
    const int fy = (int)(r % f);
    r /= f;
    const int x = (int)(r % W);
    r /= W;
    const int y = (int)(r % H);
    const int b = (int)(r / H);
    float m[9], mx = -INFINITY;
    for (int t = 0; t < 9; ++t) {
      m[t] = mask[(((size_t)b * 9 * f * f + (size_t)(t * f + fy) * f + fx) * H + y) * W + x];
      mx = fmaxf(mx, m[t]);
    }
    float den = 0.f, ux = 0.f, uy = 0.f;
    for (int t = 0; t < 9; ++t) {
      const float e = expf(m[t] - mx);
      den += e;
      const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
      if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
        ux += e * flow[((size_t)b * 2 + 0) * H * W + (size_t)yy * W + xx];
        uy += e * flow[((size_t)b * 2 + 1) * H * W + (size_t)yy * W + xx];
      }
    }
    const size_t o = ((size_t)(y * f + fy)) * (W * f) + (size_t)(x * f + fx);
    up[((size_t)b * 2 + 0) * H * W * f * f + o] = (float)f * ux / den;
    up[((size_t)b * 2 + 1) * H * W * f * f + o] = (float)f * uy / den;
  }
}

// ------------------------------------------------------------------------------------------------ resampling
// grid_sample(bilinear, padding zeros, align_corners=True) at pixel + flow: out[b, c, y, x] = in[b, c](y + fy, x + fx)
__device__ __forceinline__ float sample_zeros(const float* __restrict__ p, int H, int W, float sx, float sy) {
  const float fx0 = floorf(sx), fy0 = floorf(sy);
  const int x0 = (int)fx0, y0 = (int)fy0;
  const float ax = sx - fx0, ay = sy - fy0;
  float v = 0.f;
  if (y0 >= 0 && y0 < H) {
    if (x0 >= 0 && x0 < W) v += (1.f - ax) * (1.f - ay) * p[(size_t)y0 * W + x0];
    if (x0 + 1 >= 0 && x0 + 1 < W) v += ax * (1.f - ay) * p[(size_t)y0 * W + x0 + 1];
  }
  if (y0 + 1 >= 0 && y0 + 1 < H) {
    if (x0 >= 0 && x0 < W) v += (1.f - ax) * ay * p[(size_t)(y0 + 1) * W + x0];
    if (x0 + 1 >= 0 && x0 + 1 < W) v += ax * ay * p[(size_t)(y0 + 1) * W + x0 + 1];
  }
  return v;
}

__global__ void warp_zeros_kernel(const float* __restrict__ in, const float* __restrict__ flow, float* __restrict__ out, int B, int C,
                                  int H, int W) {
  const size_t total = (size_t)B * C * H * W;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(id % W);
    size_t r = id / W;
    const int y = (int)(r % H);
    r /= H;
    const int c = (int)(r % C);
    const int b = (int)(r / C);
    const float fx = flow[((size_t)b * 2 + 0) * H * W + (size_t)y * W + x];
    const float fy = flow[((size_t)b * 2 + 1) * H * W + (size_t)y * W + x];
    out[id] = sample_zeros(in + ((size_t)b * C + c) * H * W, H, W, (float)x + fx, (float)y + fy);
  }
}

// F.interpolate(bilinear) to (Ho, Wo), times `mul`: align_corners False (src = (dst + 0.5) * in/out - 0.5, clamped at 0) or True
__global__ void resize_bilinear_kernel(const float* __restrict__ in, float* __restrict__ out, int BC, int H, int W, int Ho, int Wo,
                                       int align, float mul) {
  const size_t total = (size_t)BC * Ho * Wo;
  const float ry = align ? (Ho > 1 ? (float)(H - 1) / (float)(Ho - 1) : 0.f) : (float)H / (float)Ho;
  const float rx = align ? (Wo > 1 ? (float)(W - 1) / (float)(Wo - 1) : 0.f) : (float)W / (float)Wo;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(id % Wo);
    size_t r = id / Wo;
    const int y = (int)(r % Ho);
    const int bc = (int)(r / Ho);
    float sy = align ? ry * (float)y : fmaxf(ry * ((float)y + 0.5f) - 0.5f, 0.f);
    float sx = align ? rx * (float)x : fmaxf(rx * ((float)x + 0.5f) - 0.5f, 0.f);
    const int y0 = min((int)sy, H - 1), x0 = min((int)sx, W - 1);
    const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
    const float ly = sy - (float)y0, lx = sx - (float)x0;
    const float* p = in + (size_t)bc * H * W;
    const float v = (1.f - ly) * ((1.f - lx) * p[(size_t)y0 * W + x0] + lx * p[(size_t)y0 * W + x1]) +
                    ly * ((1.f - lx) * p[(size_t)y1 * W + x0] + lx * p[(size_t)y1 * W + x1]);
    out[id] = v * mul;
  }
}

// MetricNet's input (MetricNet.forward :1429-1455): x = [img0 (3), img1 (3), -|img0 - warp(img1, f01)|_mean, -|img1 - warp(img0, f10)|_mean,
// f01 / ((W-1)/2, (H-1)/2) (2), f10 likewise (2), occlusion fwd, occlusion bwd] with the forward-backward check of :994-1013
__global__ void metric_input_kernel(const float* __restrict__ img0, const float* __restrict__ img1, const float* __restrict__ f01,
                                    const float* __restrict__ f10, float* __restrict__ out, int B, int H, int W) {
  const size_t total = (size_t)B * H * W, hw = (size_t)H * W;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(id % W);
    const int y = (int)((id / W) % H);
    const int b = (int)(id / hw);
    const size_t p = (size_t)y * W + x;
    const float* i0 = img0 + (size_t)b * 3 * hw;
    const float* i1 = img1 + (size_t)b * 3 * hw;
    const float* a = f01 + (size_t)b * 2 * hw;
    const float* c = f10 + (size_t)b * 2 * hw;
    const float ax = a[p], ay = a[hw + p], cx = c[p], cy = c[hw + p];
    float m0 = 0.f, m1 = 0.f;
    float* o = out + (size_t)b * 14 * hw + p;
    for (int ch = 0; ch < 3; ++ch) {
      const float v0 = i0[ch * hw + p], v1 = i1[ch * hw + p];
      m0 += fabsf(v0 - sample_zeros(i1 + ch * hw, H, W, (float)x + ax, (float)y + ay));
      m1 += fabsf(v1 - sample_zeros(i0 + ch * hw, H, W, (float)x + cx, (float)y + cy));
      o[ch * hw] = v0;
      o[(3 + ch) * hw] = v1;
    }
    o[6 * hw] = -m0 / 3.f;
    o[7 * hw] = -m1 / 3.f;
    const float nx = ((float)W - 1.f) * 0.5f, ny = ((float)H - 1.f) * 0.5f;
    o[8 * hw] = ax / nx;
    o[9 * hw] = ay / ny;
    o[10 * hw] = cx / nx;
    o[11 * hw] = cy / ny;
    // forward-backward consistency: |f + warp(b, f)| > 0.01 (|f| + |b|) + 0.5
    const float mag = sqrtf(ax * ax + ay * ay) + sqrtf(cx * cx + cy * cy);
    const float wbx = sample_zeros(c, H, W, (float)x + ax, (float)y + ay), wby = sample_zeros(c + hw, H, W, (float)x + ax, (float)y + ay);
    const float wfx = sample_zeros(a, H, W, (float)x + cx, (float)y + cy), wfy = sample_zeros(a + hw, H, W, (float)x + cx, (float)y + cy);
    const float df = sqrtf((ax + wbx) * (ax + wbx) + (ay + wby) * (ay + wby));
    const float db = sqrtf((cx + wfx) * (cx + wfx) + (cy + wfy) * (cy + wfy));
    const float thr = 0.01f * mag + 0.5f;
    o[12 * hw] = df > thr ? 1.f : 0.f;
    o[13 * hw] = db > thr ? 1.f : 0.f;
  }
}

// out[b, c, 2y + i, 2x + j] = in[b, 4c + 2i + j, y, x]
__global__ void pixel_shuffle2_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int C, int H, int W) {
  const size_t total = (size_t)B * C * 4 * H * W;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int xo = (int)(id % (2 * W));
    size_t r = id / (2 * W);
    const int yo = (int)(r % (2 * H));
    r /= 2 * H;
    const int c = (int)(r % C);
    const int b = (int)(r / C);
    out[id] = in[(((size_t)b * 4 * C + 4 * c + 2 * (yo & 1) + (xo & 1)) * H + (yo >> 1)) * W + (xo >> 1)];
  }
}

// out = post(alpha * a + beta * b + gamma), b may be null; post: 0 none, 1 relu, 2 clamp to [0, 1]; out may alias a
__global__ void axpby_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, size_t n, float alpha,
                             float beta, float gamma, int post) {
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < n; id += (size_t)gridDim.x * blockDim.x) {
    float v = alpha * a[id] + (b ? beta * b[id] : 0.f) + gamma;
    if (post == 1) v = fmaxf(v, 0.f);
    else if (post == 2) v = fminf(fmaxf(v, 0.f), 1.f);
    out[id] = v;
  }
}

// copy [B, C, H, W] into / out of a channel slice of a wider tensor, optionally cropping / zero padding the spatial size,
// optionally NHWC <-> NCHW and a per-channel affine (x - mean[c]) / std[c] (GMFlow's image normalisation)
__global__ void copy_slice_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int C, int Hs, int Ws, int Hd, int Wd,
                                  int s_ctot, int s_coff, int d_ctot, int d_coff, int src_nhwc, int dst_nhwc,
                                  const float* __restrict__ mean, const float* __restrict__ stdv) {
  const size_t total = (size_t)B * C * Hd * Wd;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(id % Wd);
    size_t r = id / Wd;
    const int y = (int)(r % Hd);
    r /= Hd;
    const int c = (int)(r % C);
    const int b = (int)(r / C);
    float v = 0.f;
    if (y < Hs && x < Ws) {
      v = src_nhwc ? src[(((size_t)b * Hs + y) * Ws + x) * s_ctot + s_coff + c]
                   : src[(((size_t)b * s_ctot + s_coff + c) * Hs + y) * Ws + x];
      if (mean) v = (v - mean[c]) / stdv[c];
    }
    if (dst_nhwc) dst[(((size_t)b * Hd + y) * Wd + x) * d_ctot + d_coff + c] = v;
    else dst[(((size_t)b * d_ctot + d_coff + c) * Hd + y) * Wd + x] = v;
  }
}

}  // namespace

#define GM_LAUNCH(kern, total, ...)                                                        \
  do {                                                                                     \
    VFI_LAUNCH(kern, grid_for_n((total), kThreads), kThreads, 0, st, __VA_ARGS__);         \
    return cudaGetLastError();                                                             \
  } while (0)

cudaError_t gm_conv2d(const float* in, const float* w, const float* bias, const float* res1, const float* res2, float* out, int N,
                      int Cin, int H, int W, int Cout, int k, int stride, int pad, int in_ctot, int in_coff, int out_ctot,
                      int out_coff, int has_pre, float pre_slope, int post, float post_slope, cudaStream_t st) {
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  const size_t total = (size_t)N * ((Cout + 15) / 16) * Ho * ((Wo + 3) / 4);
  GM_LAUNCH(conv2d_kernel, total, in, w, bias, res1, res2, out, N, Cin, H, W, Cout, Ho, Wo, k, stride, pad, in_ctot, in_coff, out_ctot,
            out_coff, has_pre, pre_slope, post, post_slope);
}
// packed form: wt [Cin * k * k][CoutP]; returns cudaErrorNotSupported for a (k, stride) the fast kernel is not built for
cudaError_t gm_conv2d_packed(const float* in, const float* wt, const float* bias, const float* res1, const float* res2, float* out,
                             int N, int Cin, int H, int W, int Cout, int CoutP, int k, int stride, int pad, int in_ctot, int in_coff,
                             int out_ctot, int out_coff, int has_pre, float pre_slope, int post, float post_slope, cudaStream_t st) {
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  const size_t total = (size_t)N * (CoutP / 16) * Ho * ((Wo + 7) / 8);
#define GM_CONV_CASE(KK, SS)                                                                                                        \
  if (k == KK && stride == SS)                                                                                                      \
    GM_LAUNCH((conv2d_packed_kernel<KK, SS>), total, in, wt, bias, res1, res2, out, N, Cin, H, W, Cout, CoutP, Ho, Wo, pad, in_ctot, \
              in_coff, out_ctot, out_coff, has_pre, pre_slope, post, post_slope)
  GM_CONV_CASE(3, 1);
  GM_CONV_CASE(3, 2);
  GM_CONV_CASE(1, 1);
  GM_CONV_CASE(1, 2);
  GM_CONV_CASE(7, 2);
#undef GM_CONV_CASE
  return cudaErrorNotSupported;
}
cudaError_t gm_convt4(const float* in, const float* w, const float* bias, float* out, int N, int Cin, int H, int W, int Cout,
                      int has_pre, float pre_slope, cudaStream_t st) {
  const size_t total = (size_t)N * ((Cout + 15) / 16) * (2 * H) * ((2 * W + 3) / 4);
  GM_LAUNCH(convt4_kernel, total, in, w, bias, out, N, Cin, H, W, Cout, has_pre, pre_slope);
}
cudaError_t gm_instance_norm(const float* in, float* out, int planes, int HW, float eps, int relu, cudaStream_t st) {
  VFI_LAUNCH(instance_norm_kernel, planes, kThreads, 0, st, in, out, HW, eps, relu);
  return cudaGetLastError();
}
cudaError_t gm_layer_norm(const float* x, const float* gamma, const float* beta, const float* src, float* out, int rows, int C,
                          float eps, cudaStream_t st) {
  VFI_LAUNCH(layer_norm_kernel, rows, kThreads, 0, st, x, gamma, beta, src, out, C, eps);
  return cudaGetLastError();
}
cudaError_t gm_softmax_rows(float* x, int rows, int L, cudaStream_t st) {
  VFI_LAUNCH(softmax_rows_kernel, rows, kThreads, 0, st, x, L);
  return cudaGetLastError();
}
cudaError_t gm_gemm(int bt, const float* A, const float* B, const float* bias, const float* mask, float* C, int nb, int M, int N, int K,
                    int lda, int ldb, int ldc, long long sA, long long sB, long long sC, float alpha, int nmask, int act,
                    cudaStream_t st) {
  const bool aligned = ((K | N | lda | ldb) & 3) == 0 && (N & 7) == 0 && ((sA | sB) & 3) == 0 &&
                       ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B)) & 15) == 0;
  if (!bt && aligned) {
    // rows per thread: 8 when that still gives the GPU enough threads, else 4 or 2 (a 7680 x 128 x 1024 linear with 8 rows
    // per thread is only 120 blocks of 8 x 8-tile threads)
    const size_t cols = (size_t)nb * (N / 8);
    const int mt = cols * ((M + 7) / 8) >= 60000 ? 8 : (cols * ((M + 3) / 4) >= 60000 ? 4 : 2);
    const size_t threads = cols * ((M + mt - 1) / mt);
    if (mt == 8) GM_LAUNCH(gemm_nn8_kernel<8>, threads, A, B, bias, mask, C, nb, M, N, K, lda, ldb, ldc, sA, sB, sC, alpha, nmask, act);
    if (mt == 4) GM_LAUNCH(gemm_nn8_kernel<4>, threads, A, B, bias, mask, C, nb, M, N, K, lda, ldb, ldc, sA, sB, sC, alpha, nmask, act);
    GM_LAUNCH(gemm_nn8_kernel<2>, threads, A, B, bias, mask, C, nb, M, N, K, lda, ldb, ldc, sA, sB, sC, alpha, nmask, act);
  }
  const size_t total = (size_t)nb * ((M + 7) / 8) * N;
  if (bt) GM_LAUNCH(gemm_kernel<true>, total, A, B, bias, mask, C, nb, M, N, K, lda, ldb, ldc, sA, sB, sC, alpha, nmask, act);
  GM_LAUNCH(gemm_kernel<false>, total, A, B, bias, mask, C, nb, M, N, K, lda, ldb, ldc, sA, sB, sC, alpha, nmask, act);
}
cudaError_t gm_transpose(const float* src, float* dst, int nb, int R, int C, cudaStream_t st) {
  GM_LAUNCH(transpose_kernel, (size_t)nb * R * C, src, dst, nb, R, C);
}
cudaError_t gm_window(const float* src, float* dst, int B, int H, int W, int C, int k, int sh, int sw, int to_windows, cudaStream_t st) {
  GM_LAUNCH(window_kernel, (size_t)B * H * W * C, src, dst, B, H, W, C, k, sh, sw, to_windows);
}
cudaError_t gm_nchw_tokens(const float* src, float* dst, int B, int C, int HW, int to_tokens, cudaStream_t st) {
  GM_LAUNCH(nchw_tokens_kernel, (size_t)B * C * HW, src, dst, B, C, HW, to_tokens);
}
cudaError_t gm_add_position(float* x, int B, int C, int H, int W, int k, cudaStream_t st) {
  GM_LAUNCH(add_position_kernel, (size_t)B * C * H * W, x, B, C, H, W, k);
}
cudaError_t gm_local_match(const float* f0, const float* f1, float* flow, int B, int C, int H, int W, int R, cudaStream_t st) {
  GM_LAUNCH(local_match_kernel, (size_t)B * H * W, f0, f1, flow, B, C, H, W, R);
}
cudaError_t gm_local_prop(const float* q, const float* k, const float* flow, float* out, int B, int C, int H, int W, cudaStream_t st) {
  GM_LAUNCH(local_prop_kernel, (size_t)B * H * W, q, k, flow, out, B, C, H, W);
}
cudaError_t gm_convex_up(const float* mask, const float* flow, float* up, int B, int H, int W, int f, cudaStream_t st) {
  GM_LAUNCH(convex_up_kernel, (size_t)B * H * W * f * f, mask, flow, up, B, H, W, f);
}
cudaError_t gm_warp_zeros(const float* in, const float* flow, float* out, int B, int C, int H, int W, cudaStream_t st) {
  GM_LAUNCH(warp_zeros_kernel, (size_t)B * C * H * W, in, flow, out, B, C, H, W);
}
cudaError_t gm_resize(const float* in, float* out, int BC, int H, int W, int Ho, int Wo, int align, float mul, cudaStream_t st) {
  GM_LAUNCH(resize_bilinear_kernel, (size_t)BC * Ho * Wo, in, out, BC, H, W, Ho, Wo, align, mul);
}
cudaError_t gm_metric_input(const float* img0, const float* img1, const float* f01, const float* f10, float* out, int B, int H, int W,
                            cudaStream_t st) {
  GM_LAUNCH(metric_input_kernel, (size_t)B * H * W, img0, img1, f01, f10, out, B, H, W);
}
cudaError_t gm_pixel_shuffle2(const float* in, float* out, int B, int C, int H, int W, cudaStream_t st) {
  GM_LAUNCH(pixel_shuffle2_kernel, (size_t)B * C * 4 * H * W, in, out, B, C, H, W);
}
cudaError_t gm_axpby(const float* a, const float* b, float* out, size_t n, float alpha, float beta, float gamma, int post,
                     cudaStream_t st) {
  GM_LAUNCH(axpby_kernel, n, a, b, out, n, alpha, beta, gamma, post);
}
cudaError_t gm_copy_slice(const float* src, float* dst, int B, int C, int Hs, int Ws, int Hd, int Wd, int s_ctot, int s_coff, int d_ctot,
                          int d_coff, int src_nhwc, int dst_nhwc, const float* mean, const float* stdv, cudaStream_t st) {
  GM_LAUNCH(copy_slice_kernel, (size_t)B * C * Hd * Wd, src, dst, B, C, Hs, Ws, Hd, Wd, s_ctot, s_coff, d_ctot, d_coff, src_nhwc, dst_nhwc,
            mean, stdv);
}

}  // namespace vfi

// =================================================================================================
// C ABI (include/vfi_b200.h): thin argument checks around the launchers; DEVICE pointers, fp32, caller's stream
// =================================================================================================
namespace {
int gm_fail(const char* what) {
  vfi::set_error(std::string("vfi_gm: ") + what);
  return VFI_E_INVALID;
}
int gm_done(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return VFI_OK;
  vfi::set_error(std::string("vfi_gm_") + what + ": " + cudaGetErrorString(e));
  return VFI_E_CUDA;
}
}  // namespace

extern "C" {

int vfi_gm_conv2d(const float* in, const float* w, const float* bias, const float* res1, const float* res2, float* out, int N, int Cin,
                  int H, int W, int Cout, int k, int stride, int pad, int in_ctot, int in_coff, int out_ctot, int out_coff, int has_pre,
                  float pre_slope, int post, float post_slope, void* stream) {
  if (!in || !w || !out || N < 1 || Cin < 1 || Cout < 1 || H < 1 || W < 1 || k < 1 || stride < 1 || pad < 0) return gm_fail("conv2d: bad argument");
  if (in_coff < 0 || in_coff + Cin > in_ctot || out_coff < 0 || out_coff + Cout > out_ctot) return gm_fail("conv2d: channel slice out of range");
  return gm_done(vfi::gm_conv2d(in, w, bias, res1, res2, out, N, Cin, H, W, Cout, k, stride, pad, in_ctot, in_coff, out_ctot, out_coff,
                                has_pre, pre_slope, post, post_slope, (cudaStream_t)stream), "conv2d");
}
int vfi_gm_conv2d_packed(const float* in, const float* wt, const float* bias, const float* res1, const float* res2, float* out, int N,
                         int Cin, int H, int W, int Cout, int CoutP, int k, int stride, int pad, int in_ctot, int in_coff, int out_ctot,
                         int out_coff, int has_pre, float pre_slope, int post, float post_slope, void* stream) {
  if (!in || !wt || !out || N < 1 || Cin < 1 || Cout < 1 || CoutP < Cout || (CoutP & 15) || H < 1 || W < 1 || pad < 0 ||
      (reinterpret_cast<uintptr_t>(wt) & 15))
    return gm_fail("conv2d_packed: bad argument");
  if (in_coff < 0 || in_coff + Cin > in_ctot || out_coff < 0 || out_coff + Cout > out_ctot) return gm_fail("conv2d_packed: channel slice out of range");
  if (!((k == 3 || k == 1) && (stride == 1 || stride == 2)) && !(k == 7 && stride == 2)) return gm_fail("conv2d_packed: kernel size / stride not built");
  return gm_done(vfi::gm_conv2d_packed(in, wt, bias, res1, res2, out, N, Cin, H, W, Cout, CoutP, k, stride, pad, in_ctot, in_coff, out_ctot,
                                       out_coff, has_pre, pre_slope, post, post_slope, (cudaStream_t)stream), "conv2d_packed");
}
int vfi_gm_transpose(const float* src, float* dst, int nb, int R, int C, void* stream) {
  if (!src || !dst || nb < 1 || R < 1 || C < 1) return gm_fail("transpose: bad argument");
  return gm_done(vfi::gm_transpose(src, dst, nb, R, C, (cudaStream_t)stream), "transpose");
}
int vfi_gm_convt4(const float* in, const float* w, const float* bias, float* out, int N, int Cin, int H, int W, int Cout, int has_pre,
                  float pre_slope, void* stream) {
  if (!in || !w || !out || N < 1 || Cin < 1 || Cout < 1 || H < 1 || W < 1) return gm_fail("convt4: bad argument");
  return gm_done(vfi::gm_convt4(in, w, bias, out, N, Cin, H, W, Cout, has_pre, pre_slope, (cudaStream_t)stream), "convt4");
}
int vfi_gm_instance_norm(const float* in, float* out, int planes, int HW, float eps, int relu, void* stream) {
  if (!in || !out || planes < 1 || HW < 1) return gm_fail("instance_norm: bad argument");
  return gm_done(vfi::gm_instance_norm(in, out, planes, HW, eps, relu, (cudaStream_t)stream), "instance_norm");
}
int vfi_gm_layer_norm(const float* x, const float* gamma, const float* beta, const float* src, float* out, int rows, int C, float eps,
                      void* stream) {
  if (!x || !gamma || !beta || !out || rows < 1 || C < 1) return gm_fail("layer_norm: bad argument");
  return gm_done(vfi::gm_layer_norm(x, gamma, beta, src, out, rows, C, eps, (cudaStream_t)stream), "layer_norm");
}
int vfi_gm_softmax_rows(float* x, int rows, int L, void* stream) {
  if (!x || rows < 1 || L < 1) return gm_fail("softmax_rows: bad argument");
  return gm_done(vfi::gm_softmax_rows(x, rows, L, (cudaStream_t)stream), "softmax_rows");
}
int vfi_gm_gemm(int bt, const float* A, const float* B, const float* bias, const float* mask, float* C, int nb, int M, int N, int K,
                int lda, int ldb, int ldc, long long sA, long long sB, long long sC, float alpha, int nmask, int act, void* stream) {
  if (!A || !B || !C || nb < 1 || M < 1 || N < 1 || K < 1 || (mask && nmask < 1)) return gm_fail("gemm: bad argument");
  return gm_done(vfi::gm_gemm(bt, A, B, bias, mask, C, nb, M, N, K, lda, ldb, ldc, sA, sB, sC, alpha, nmask, act, (cudaStream_t)stream), "gemm");
}
int vfi_gm_window(const float* src, float* dst, int B, int H, int W, int C, int k, int sh, int sw, int to_windows, void* stream) {
  if (!src || !dst || B < 1 || H < 1 || W < 1 || C < 1 || k < 1 || H % k || W % k) return gm_fail("window: bad argument");
  return gm_done(vfi::gm_window(src, dst, B, H, W, C, k, sh, sw, to_windows, (cudaStream_t)stream), "window");
}
int vfi_gm_nchw_tokens(const float* src, float* dst, int B, int C, int HW, int to_tokens, void* stream) {
  if (!src || !dst || B < 1 || C < 1 || HW < 1) return gm_fail("nchw_tokens: bad argument");
  return gm_done(vfi::gm_nchw_tokens(src, dst, B, C, HW, to_tokens, (cudaStream_t)stream), "nchw_tokens");
}
int vfi_gm_add_position(float* x, int B, int C, int H, int W, int k, void* stream) {
  if (!x || B < 1 || C < 2 || (C & 1) || H < 1 || W < 1 || k < 1 || H % k || W % k) return gm_fail("add_position: bad argument");
  return gm_done(vfi::gm_add_position(x, B, C, H, W, k, (cudaStream_t)stream), "add_position");
}
int vfi_gm_local_match(const float* f0, const float* f1, float* flow, int B, int C, int H, int W, int R, void* stream) {
  if (!f0 || !f1 || !flow || B < 1 || C < 1 || H < 1 || W < 1 || R < 1 || R > 4) return gm_fail("local_match: bad argument");
  return gm_done(vfi::gm_local_match(f0, f1, flow, B, C, H, W, R, (cudaStream_t)stream), "local_match");
}
int vfi_gm_local_prop(const float* q, const float* k, const float* flow, float* out, int B, int C, int H, int W, void* stream) {
  if (!q || !k || !flow || !out || B < 1 || C < 1 || H < 1 || W < 1) return gm_fail("local_prop: bad argument");
  return gm_done(vfi::gm_local_prop(q, k, flow, out, B, C, H, W, (cudaStream_t)stream), "local_prop");
}
int vfi_gm_convex_up(const float* mask, const float* flow, float* up, int B, int H, int W, int f, void* stream) {
  if (!mask || !flow || !up || B < 1 || H < 1 || W < 1 || f < 1) return gm_fail("convex_up: bad argument");
  return gm_done(vfi::gm_convex_up(mask, flow, up, B, H, W, f, (cudaStream_t)stream), "convex_up");
}
int vfi_gm_warp_zeros(const float* in, const float* flow, float* out, int B, int C, int H, int W, void* stream) {
  if (!in || !flow || !out || B < 1 || C < 1 || H < 1 || W < 1) return gm_fail("warp_zeros: bad argument");
  return gm_done(vfi::gm_warp_zeros(in, flow, out, B, C, H, W, (cudaStream_t)stream), "warp_zeros");
}
int vfi_gm_resize(const float* in, float* out, int BC, int H, int W, int Ho, int Wo, int align, float mul, void* stream) {
  if (!in || !out || BC < 1 || H < 1 || W < 1 || Ho < 1 || Wo < 1) return gm_fail("resize: bad argument");
  return gm_done(vfi::gm_resize(in, out, BC, H, W, Ho, Wo, align, mul, (cudaStream_t)stream), "resize");
}
int vfi_gm_metric_input(const float* img0, const float* img1, const float* f01, const float* f10, float* out, int B, int H, int W,
                        void* stream) {
  if (!img0 || !img1 || !f01 || !f10 || !out || B < 1 || H < 2 || W < 2) return gm_fail("metric_input: bad argument");
  return gm_done(vfi::gm_metric_input(img0, img1, f01, f10, out, B, H, W, (cudaStream_t)stream), "metric_input");
}
int vfi_gm_pixel_shuffle2(const float* in, float* out, int B, int C, int H, int W, void* stream) {
  if (!in || !out || B < 1 || C < 1 || H < 1 || W < 1) return gm_fail("pixel_shuffle2: bad argument");
  return gm_done(vfi::gm_pixel_shuffle2(in, out, B, C, H, W, (cudaStream_t)stream), "pixel_shuffle2");
}
int vfi_gm_axpby(const float* a, const float* b, float* out, long long n, float alpha, float beta, float gamma, int post, void* stream) {
  if (!a || !out || n < 1) return gm_fail("axpby: bad argument");
  return gm_done(vfi::gm_axpby(a, b, out, (size_t)n, alpha, beta, gamma, post, (cudaStream_t)stream), "axpby");
}
int vfi_gm_copy_slice(const float* src, float* dst, int B, int C, int Hs, int Ws, int Hd, int Wd, int s_ctot, int s_coff, int d_ctot,
                      int d_coff, int src_nhwc, int dst_nhwc, const float* mean, const float* stdv, void* stream) {
  if (!src || !dst || B < 1 || C < 1 || Hs < 1 || Ws < 1 || Hd < 1 || Wd < 1 || s_coff < 0 || d_coff < 0 || s_coff + C > s_ctot ||
      d_coff + C > d_ctot || ((mean == nullptr) != (stdv == nullptr)))
    return gm_fail("copy_slice: bad argument");
  return gm_done(vfi::gm_copy_slice(src, dst, B, C, Hs, Ws, Hd, Wd, s_ctot, s_coff, d_ctot, d_coff, src_nhwc, dst_nhwc, mean, stdv,
                                    (cudaStream_t)stream), "copy_slice");
}

}  // extern "C"
