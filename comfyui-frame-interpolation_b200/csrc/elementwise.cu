// Full-resolution, HBM-bound kernels of the RIFE-4.6 path (fp32 flow / mask / image arithmetic):
//   prep_frames : clamp(0,1) + zero-pad to x64 + RGB->float4           rife_arch.py:476-485
//   front       : [warp(img0), warp(img1), t, mask, flow] -> bilinear 1/s -> 16-channel block input, written
//                 directly in the space-to-depth form the stride-2 conv0.0 reads
//                                                                       rife_arch.py:31-70, :238-249, :589-596
//   (flow)      : flow = sum_j up_sj(T_j)*s_j is evaluated on the fly from the blocks' low-res outputs   rife_arch.py:263-266, :694-696
//   final       : warp both frames with the final flow, sigmoid blend, crop, clamp    rife_arch.py:703-704, :713-717, :732
//   warp        : stand-alone backward bilinear warp (border, align_corners=True), NHWC fp32, any C
#include "ptx.cuh"
#include "vfi_internal.h"

namespace vfi {
namespace {

__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

__global__ void prep_frames_kernel(const float* __restrict__ frames, int n, int H, int W, int cstride,
                                   float4* __restrict__ imgs, uint2* __restrict__ imgs_h, int Hp, int Wp) {
  const size_t total = (size_t)n * Hp * Wp;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(id % Wp);
    const size_t r = id / Wp;
    const int y = (int)(r % Hp);
    const int f = (int)(r / Hp);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (y < H && x < W) {
      const float* s = frames + (((size_t)f * H + y) * W + x) * cstride;
      v.x = clamp01(__ldg(s));
      v.y = clamp01(__ldg(s + 1));
      v.z = clamp01(__ldg(s + 2));
    }
    imgs[id] = v;
    imgs_h[id] = make_uint2(Pack2<__half>::pack(v.x, v.y), Pack2<__half>::pack(v.z, 0.f));
  }
}

// half4 pixel -> float4
__device__ __forceinline__ float4 unpack_h4(uint2 q) {
  const float2 a = Pack2<__half>::unpack(q.x), b = Pack2<__half>::unpack(q.y);
  return make_float4(a.x, a.y, b.x, b.y);
}

// grid_sample(bilinear, border, align_corners=True) at (x + fx, y + fy) of a float4 image [Hp][Wp]
__device__ __forceinline__ float4 sample_border(const float4* __restrict__ img, int Hp, int Wp, float sx, float sy) {
  sx = fminf(fmaxf(sx, 0.f), (float)(Wp - 1));
  sy = fminf(fmaxf(sy, 0.f), (float)(Hp - 1));
  const float fx0 = floorf(sx), fy0 = floorf(sy);
  const int x0 = (int)fx0, y0 = (int)fy0;
  const int dx = (x0 + 1 < Wp) ? 1 : 0, dyw = (y0 + 1 < Hp) ? Wp : 0;  // x1 = min(x0+1, Wp-1), y1 likewise
  const float ax = sx - fx0, ay = sy - fy0;
  const float w00 = (1.f - ax) * (1.f - ay), w01 = ax * (1.f - ay), w10 = (1.f - ax) * ay, w11 = ax * ay;
  const float4* p = img + (y0 * Wp + x0);  // one plane is < 2^31 pixels: 32-bit offsets
  const float4 a = __ldg(p);
  const float4 b = __ldg(p + dx);
  const float4 c = __ldg(p + dyw);
  const float4 d = __ldg(p + dyw + dx);
  float4 o;
  o.x = a.x * w00 + b.x * w01 + c.x * w10 + d.x * w11;
  o.y = a.y * w00 + b.y * w01 + c.y * w10 + d.y * w11;
  o.z = a.z * w00 + b.z * w01 + c.z * w10 + d.z * w11;
  o.w = 0.f;
  return o;
}

// the same sampling of a half4 image plane (block inputs; interpolation in fp32)
__device__ __forceinline__ float4 sample_border(const uint2* __restrict__ img, int Hp, int Wp, float sx, float sy) {
  sx = fminf(fmaxf(sx, 0.f), (float)(Wp - 1));
  sy = fminf(fmaxf(sy, 0.f), (float)(Hp - 1));
  const float fx0 = floorf(sx), fy0 = floorf(sy);
  const int x0 = (int)fx0, y0 = (int)fy0;
  const int dx = (x0 + 1 < Wp) ? 1 : 0, dyw = (y0 + 1 < Hp) ? Wp : 0;
  const float ax = sx - fx0, ay = sy - fy0;
  const float w00 = (1.f - ax) * (1.f - ay), w01 = ax * (1.f - ay), w10 = (1.f - ax) * ay, w11 = ax * ay;
  const uint2* p = img + (y0 * Wp + x0);
  const float4 a = unpack_h4(__ldg(p));
  const float4 b = unpack_h4(__ldg(p + dx));
  const float4 c = unpack_h4(__ldg(p + dyw));
  const float4 d = unpack_h4(__ldg(p + dyw + dx));
  float4 o;
  o.x = a.x * w00 + b.x * w01 + c.x * w10 + d.x * w11;
  o.y = a.y * w00 + b.y * w01 + c.y * w10 + d.y * w11;
  o.z = a.z * w00 + b.z * w01 + c.z * w10 + d.z * w11;
  o.w = 0.f;
  return o;
}

// same sampling for a 4-channel feature plane (arch 4.7 encode features, stored as half4)
__device__ __forceinline__ float4 sample_border4(const uint2* __restrict__ img, int Hp, int Wp, float sx, float sy) {
  sx = fminf(fmaxf(sx, 0.f), (float)(Wp - 1));
  sy = fminf(fmaxf(sy, 0.f), (float)(Hp - 1));
  const float fx0 = floorf(sx), fy0 = floorf(sy);
  const int x0 = (int)fx0, y0 = (int)fy0;
  const int dx = (x0 + 1 < Wp) ? 1 : 0, dyw = (y0 + 1 < Hp) ? Wp : 0;
  const float ax = sx - fx0, ay = sy - fy0;
  const float w00 = (1.f - ax) * (1.f - ay), w01 = ax * (1.f - ay), w10 = (1.f - ax) * ay, w11 = ax * ay;
  const uint2* p = img + (y0 * Wp + x0);
  const float4 a = unpack_h4(__ldg(p));
  const float4 b = unpack_h4(__ldg(p + dx));
  const float4 c = unpack_h4(__ldg(p + dyw));
  const float4 d = unpack_h4(__ldg(p + dyw + dx));
  float4 o;
  o.x = a.x * w00 + b.x * w01 + c.x * w10 + d.x * w11;
  o.y = a.y * w00 + b.y * w01 + c.y * w10 + d.y * w11;
  o.z = a.z * w00 + b.z * w01 + c.z * w10 + d.z * w11;
  o.w = a.w * w00 + b.w * w01 + c.w * w10 + d.w * w11;
  return o;
}

// ---------------------------------------------------------------------------------------------
// Flow state.  The reference keeps flow/mask at full resolution and adds each block's up-scaled output to it
// (rife_arch.py:263-266, :694-696).  Here each block leaves only its low-resolution output T_j (float4 flow +
// float mask at 1/s_j) and the consumers evaluate
//      flow(p) = base(p) + sum_j up(T_j)(p) * s_j          (same fp32 summation order as the reference)
// where `base` is a full-resolution plane that is written only by a front kernel that visits every pixel anyway
// (s <= 2), never by a separate pass: with scales 8,4,2,1  block 1 reads {T0}, block 2 reads {T0,T1} and stores
// F1, block 3 reads F1+{T2} and stores F2, the final blend reads F2+{T3}.  (A fully implicit variant needs 24 extra
// loads per pixel in block 3, and a separate up-sample/accumulate pass per block moves 2x the bytes.)
// ---------------------------------------------------------------------------------------------
struct FlowLevels {
  const float4* f[kMaxBlocks];  // levels to add, in order: [B, Hp/s, Wp/s] flow increments
  const float* m[kMaxBlocks];   //                          [B, Hp/s, Wp/s] mask increments
  int s[kMaxBlocks];
  int hs[kMaxBlocks], ws[kMaxBlocks];  // level size Hp/s, Wp/s (set by the host: no integer division in the kernels)
  float inv_s[kMaxBlocks];             // 1/s
  const float4* base_f;  // optional full-resolution accumulated flow [B, Hp, Wp] (nullptr: start from zero)
  const float* base_m;
  float4* out_f;         // optional: store the accumulated flow / mask at every visited position
  float* out_m;
  int mask_replace;      // arch 4.7+: mask = the newest level's mask (rife_arch.py:698-699), not the running sum
};

// F.interpolate(scale_factor=s, bilinear, align_corners=False) of level j at full-res position (Y, X)
__device__ __forceinline__ void up_level(const FlowLevels& L, int j, int b, int Hp, int Wp, int Y, int X, float4& uf,
                                         float& um) {
  const int s = L.s[j];
  const int Hs = L.hs[j], Ws = L.ws[j];
  const float4* tf = L.f[j] + (size_t)b * Hs * Ws;
  const float* tm = L.m[j] + (size_t)b * Hs * Ws;
  if (s == 1) {
    uf = __ldg(tf + (Y * Ws + X));
    um = __ldg(tm + (Y * Ws + X));
    return;
  }
  const float inv_s = L.inv_s[j];
  const float sy = fmaxf(((float)Y + 0.5f) * inv_s - 0.5f, 0.f);
  const float sx = fmaxf(((float)X + 0.5f) * inv_s - 0.5f, 0.f);
  const int y0 = min((int)sy, Hs - 1), x0 = min((int)sx, Ws - 1);
  const int dx = (x0 + 1 < Ws) ? 1 : 0, dyw = (y0 + 1 < Hs) ? Ws : 0;  // x1 = min(x0+1, Ws-1), y1 likewise
  const float ly = sy - (float)y0, lx = sx - (float)x0;
  const float hy = 1.f - ly, hx = 1.f - lx;
  const int o00 = y0 * Ws + x0;  // one level plane is < 2^31 elements
  const float4 a = __ldg(tf + o00);
  const float4 bq = __ldg(tf + o00 + dx);
  const float4 c = __ldg(tf + o00 + dyw);
  const float4 d = __ldg(tf + o00 + dyw + dx);
  const float ma = __ldg(tm + o00);
  const float mb = __ldg(tm + o00 + dx);
  const float mc = __ldg(tm + o00 + dyw);
  const float md = __ldg(tm + o00 + dyw + dx);
  uf.x = hy * (hx * a.x + lx * bq.x) + ly * (hx * c.x + lx * d.x);
  uf.y = hy * (hx * a.y + lx * bq.y) + ly * (hx * c.y + lx * d.y);
  uf.z = hy * (hx * a.z + lx * bq.z) + ly * (hx * c.z + lx * d.z);
  uf.w = hy * (hx * a.w + lx * bq.w) + ly * (hx * c.w + lx * d.w);
  um = hy * (hx * ma + lx * mb) + ly * (hx * mc + lx * md);
}

// accumulated flow / mask at a full-resolution position, in the reference's summation order
template <int NLEV>
__device__ __forceinline__ void flow_at(const FlowLevels& L, int b, int Hp, int Wp, int Y, int X, float4& f,
                                        float& m) {
  const size_t pid = ((size_t)b * Hp + Y) * Wp + X;
  float4 u;
  float um;
  if (L.base_f != nullptr) {
    f = L.base_f[pid];  // plain loads: the same thread may store the updated value to this address below
    m = L.base_m[pid];
  } else {
    up_level(L, 0, b, Hp, Wp, Y, X, u, um);
    const float s0 = (float)L.s[0];
    f = make_float4(u.x * s0, u.y * s0, u.z * s0, u.w * s0);
    m = um;
  }
#pragma unroll
  for (int j = 0; j < NLEV; ++j) {
    if (j == 0 && L.base_f == nullptr) continue;
    up_level(L, j, b, Hp, Wp, Y, X, u, um);
    const float sj = (float)L.s[j];
    f.x += u.x * sj;
    f.y += u.y * sj;
    f.z += u.z * sj;
    f.w += u.w * sj;
    m = L.mask_replace ? um : m + um;
  }
  if (L.out_f != nullptr) {
    L.out_f[pid] = f;
    L.out_m[pid] = m;
  }
}

// one thread = one cell of the 1/s grid; channels: w0.rgb, w1.rgb, t, mask, flow/s (4) [, 4 zero pad].
// Thread order (b, row pair, x, row parity) so that 4 consecutive lanes fill one 128-byte space-to-depth cell.
template <typename T, int NLEV, int S>
__global__ void front_kernel(const uint2* __restrict__ imgs, const FlowLevels lev, const BatchTasks tasks, int Hp,
                             int Wp, int s_rt, T* __restrict__ x_s2d) {
  const int s = S ? S : s_rt;
  const int Hs = Hp / s, Ws = Wp / s;
  const size_t plane = (size_t)Hp * Wp;
  const float inv_s = 1.f / (float)s;
  // grid = (x cells / 64, row pairs, images): no 64-bit integer division of a flat index per thread
  {
    const int par = (int)(threadIdx.x & 1);
    const int xl = (int)(blockIdx.x * (blockDim.x >> 1) + (threadIdx.x >> 1));
    if (xl >= Ws) return;
    const int yl = (int)blockIdx.y * 2 + par;
    const int b = (int)blockIdx.z;
    const uint2* img0 = imgs + (size_t)tasks.f0[b] * plane;
    const uint2* img1 = imgs + (size_t)tasks.f1[b] * plane;
    const float t = tasks.t[b];
    // bilinear 1/s, align_corners=False: the two source taps per axis are s*i + s/2 - 1 and s*i + s/2, weight 1/2
    const int ntap = (s == 1) ? 1 : 2;
    const int by = (s == 1) ? yl : s * yl + s / 2 - 1;
    const int bx = (s == 1) ? xl : s * xl + s / 2 - 1;
    float ch[12];
    float rowacc[2][12];
#pragma unroll
    for (int ty = 0; ty < 2; ++ty) {
      float colv[2][12];
#pragma unroll
      for (int tx = 0; tx < 2; ++tx) {
        if (ty < ntap && tx < ntap) {
          const int Y = by + ty, X = bx + tx;
          float* v = colv[tx];
          if (NLEV == 0) {
            const float4 a = unpack_h4(__ldg(img0 + (size_t)Y * Wp + X));
            const float4 c = unpack_h4(__ldg(img1 + (size_t)Y * Wp + X));
            v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = c.x; v[4] = c.y; v[5] = c.z;
            v[6] = t; v[7] = 0.f; v[8] = 0.f; v[9] = 0.f; v[10] = 0.f; v[11] = 0.f;
          } else {
            float4 f;
            float m;
            flow_at<(NLEV > 0 ? NLEV : 1)>(lev, b, Hp, Wp, Y, X, f, m);
            const float4 a = sample_border(img0, Hp, Wp, (float)X + f.x, (float)Y + f.y);
            const float4 c = sample_border(img1, Hp, Wp, (float)X + f.z, (float)Y + f.w);
            v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = c.x; v[4] = c.y; v[5] = c.z;
            v[6] = t; v[7] = m; v[8] = f.x; v[9] = f.y; v[10] = f.z; v[11] = f.w;
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 12; ++i) rowacc[ty][i] = (ntap == 1) ? colv[0][i] : (colv[0][i] + colv[1][i]);
    }
#pragma unroll
    for (int i = 0; i < 12; ++i) ch[i] = (ntap == 1) ? rowacc[0][i] : 0.25f * (rowacc[0][i] + rowacc[1][i]);
#pragma unroll
    for (int i = 8; i < 12; ++i) ch[i] *= inv_s;  // flow is also divided by the scale (rife_arch.py:242-248)

    // space-to-depth store: cell (yl, xl) -> [b, yl/2, xl/2, ((yl&1)*2 + (xl&1))*16 + c]
    const size_t cell = ((size_t)b * (Hs >> 1) + (yl >> 1)) * (Ws >> 1) + (xl >> 1);
    T* dst = x_s2d + cell * 64 + ((yl & 1) * 2 + (xl & 1)) * 16;
    uint4 lo, hi;
    lo.x = Pack2<T>::pack(ch[0], ch[1]);
    lo.y = Pack2<T>::pack(ch[2], ch[3]);
    lo.z = Pack2<T>::pack(ch[4], ch[5]);
    lo.w = Pack2<T>::pack(ch[6], ch[7]);
    hi.x = Pack2<T>::pack(ch[8], ch[9]);
    hi.y = Pack2<T>::pack(ch[10], ch[11]);
    hi.z = 0u;
    hi.w = 0u;
    reinterpret_cast<uint4*>(dst)[0] = lo;
    reinterpret_cast<uint4*>(dst)[1] = hi;
  }
}


// ---- scale-2 front with shared level taps ---------------------------------------------------------------------
// The four full-resolution pixels (2yl+ty, 2xl+tx) of one half-resolution cell fall between the same 2x2 samples of
// every coarser level (scale s_l = 4, 8, ...: an integer sample boundary u = n would need s_l(n + 1/2) = 2xl + 1,
// even = odd), so the level taps are loaded once per cell and only the bilinear weights differ per pixel.  Same
// arithmetic per pixel as up_level()/flow_at().
struct LevelTap {
  float4 a, b, c, d;
  float ma, mb, mc, md;
  float fy0, fx0, inv_s, sc;
};

__device__ __forceinline__ void load_level_tap(const FlowLevels& L, int j, int b, int Hp, int Wp, int Y0, int X0,
                                               LevelTap& t) {
  const int Hs = L.hs[j], Ws = L.ws[j];
  const float4* tf = L.f[j] + (size_t)b * Hs * Ws;
  const float* tm = L.m[j] + (size_t)b * Hs * Ws;
  t.inv_s = L.inv_s[j];
  t.sc = (float)L.s[j];
  const float sy = fmaxf(((float)Y0 + 0.5f) * t.inv_s - 0.5f, 0.f);
  const float sx = fmaxf(((float)X0 + 0.5f) * t.inv_s - 0.5f, 0.f);
  const int y0 = min((int)sy, Hs - 1), x0 = min((int)sx, Ws - 1);
  const int dx = (x0 + 1 < Ws) ? 1 : 0, dyw = (y0 + 1 < Hs) ? Ws : 0;
  t.fy0 = (float)y0;
  t.fx0 = (float)x0;
  const int o00 = y0 * Ws + x0;
  t.a = __ldg(tf + o00);
  t.b = __ldg(tf + o00 + dx);
  t.c = __ldg(tf + o00 + dyw);
  t.d = __ldg(tf + o00 + dyw + dx);
  t.ma = __ldg(tm + o00);
  t.mb = __ldg(tm + o00 + dx);
  t.mc = __ldg(tm + o00 + dyw);
  t.md = __ldg(tm + o00 + dyw + dx);
}

__device__ __forceinline__ void eval_level_tap(const LevelTap& t, int Y, int X, float4& uf, float& um) {
  const float sy = fmaxf(((float)Y + 0.5f) * t.inv_s - 0.5f, 0.f);
  const float sx = fmaxf(((float)X + 0.5f) * t.inv_s - 0.5f, 0.f);
  const float ly = sy - t.fy0, lx = sx - t.fx0;
  const float hy = 1.f - ly, hx = 1.f - lx;
  uf.x = hy * (hx * t.a.x + lx * t.b.x) + ly * (hx * t.c.x + lx * t.d.x);
  uf.y = hy * (hx * t.a.y + lx * t.b.y) + ly * (hx * t.c.y + lx * t.d.y);
  uf.z = hy * (hx * t.a.z + lx * t.b.z) + ly * (hx * t.c.z + lx * t.d.z);
  uf.w = hy * (hx * t.a.w + lx * t.b.w) + ly * (hx * t.c.w + lx * t.d.w);
  um = hy * (hx * t.ma + lx * t.mb) + ly * (hx * t.mc + lx * t.md);
}

// one thread = one half-resolution cell, no base plane (the first dense front), levels 0..NLEV-1 all of scale >= 4
template <typename T, int NLEV>
__global__ void front2_kernel(const uint2* __restrict__ imgs, const FlowLevels lev, const BatchTasks tasks, int Hp,
                              int Wp, T* __restrict__ x_s2d) {
  const int Hs = Hp >> 1, Ws = Wp >> 1;
  const size_t plane = (size_t)Hp * Wp;
  {
    const int par = (int)(threadIdx.x & 1);
    const int xl = (int)(blockIdx.x * (blockDim.x >> 1) + (threadIdx.x >> 1));
    if (xl >= Ws) return;
    const int yl = (int)blockIdx.y * 2 + par;
    const int b = (int)blockIdx.z;
    const uint2* img0 = imgs + (size_t)tasks.f0[b] * plane;
    const uint2* img1 = imgs + (size_t)tasks.f1[b] * plane;
    const int Y0 = 2 * yl, X0 = 2 * xl;
    float4 f[4];
    float m[4];
#pragma unroll
    for (int j = 0; j < NLEV; ++j) {
      LevelTap tp;
      load_level_tap(lev, j, b, Hp, Wp, Y0, X0, tp);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float4 u;
        float um;
        eval_level_tap(tp, Y0 + (q >> 1), X0 + (q & 1), u, um);
        if (j == 0) {
          f[q] = make_float4(u.x * tp.sc, u.y * tp.sc, u.z * tp.sc, u.w * tp.sc);
          m[q] = um;
        } else {
          f[q].x += u.x * tp.sc;
          f[q].y += u.y * tp.sc;
          f[q].z += u.z * tp.sc;
          f[q].w += u.w * tp.sc;
          m[q] = lev.mask_replace ? um : m[q] + um;
        }
      }
    }
    float ch[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) ch[i] = 0.f;
    // same summation order as the generic kernel: (tap00 + tap01) + (tap10 + tap11), then * 0.25
    float row[2][12];
#pragma unroll
    for (int ty = 0; ty < 2; ++ty) {
      float v[2][12];
#pragma unroll
      for (int tx = 0; tx < 2; ++tx) {
        const int q = ty * 2 + tx;
        const int Y = Y0 + ty, X = X0 + tx;
        const float4 a = sample_border(img0, Hp, Wp, (float)X + f[q].x, (float)Y + f[q].y);
        const float4 c = sample_border(img1, Hp, Wp, (float)X + f[q].z, (float)Y + f[q].w);
        v[tx][0] = a.x; v[tx][1] = a.y; v[tx][2] = a.z; v[tx][3] = c.x; v[tx][4] = c.y; v[tx][5] = c.z;
        v[tx][6] = tasks.t[b]; v[tx][7] = m[q];
        v[tx][8] = f[q].x; v[tx][9] = f[q].y; v[tx][10] = f[q].z; v[tx][11] = f[q].w;
      }
#pragma unroll
      for (int i = 0; i < 12; ++i) row[ty][i] = v[0][i] + v[1][i];
    }
#pragma unroll
    for (int i = 0; i < 12; ++i) ch[i] = 0.25f * (row[0][i] + row[1][i]);
#pragma unroll
    for (int i = 8; i < 12; ++i) ch[i] *= 0.5f;
    if (lev.out_f != nullptr) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const size_t pid = ((size_t)b * Hp + Y0 + (q >> 1)) * Wp + X0 + (q & 1);
        lev.out_f[pid] = f[q];
        lev.out_m[pid] = m[q];
      }
    }
    const size_t cell = ((size_t)b * (Hs >> 1) + (yl >> 1)) * (Ws >> 1) + (xl >> 1);
    T* dst = x_s2d + cell * 64 + ((yl & 1) * 2 + (xl & 1)) * 16;
    uint4 lo, hi;
    lo.x = Pack2<T>::pack(ch[0], ch[1]);
    lo.y = Pack2<T>::pack(ch[2], ch[3]);
    lo.z = Pack2<T>::pack(ch[4], ch[5]);
    lo.w = Pack2<T>::pack(ch[6], ch[7]);
    hi.x = Pack2<T>::pack(ch[8], ch[9]);
    hi.y = Pack2<T>::pack(ch[10], ch[11]);
    hi.z = 0u;
    hi.w = 0u;
    reinterpret_cast<uint4*>(dst)[0] = lo;
    reinterpret_cast<uint4*>(dst)[1] = hi;
  }
}

// ---------------------------------------------------------------------------------------------
// arch 4.7 (rife47.pth / rife49.pth): encode head  f = ConvTranspose2d(16,4,4,2,1)(Conv2d(3,16,3,2,1)(img))
// (rife_arch.py:414-416, :501-503), once per source frame, fp32 on the CUDA cores (0.76 GMAC per 1080p frame).
// ---------------------------------------------------------------------------------------------
__global__ void encode_conv_kernel(const float4* __restrict__ imgs, const float* __restrict__ w,
                                   const float* __restrict__ bias, float* __restrict__ e16, int n, int Hp, int Wp) {
  __shared__ float ws[16 * 27 + 16];
  for (int i = threadIdx.x; i < 16 * 27; i += blockDim.x) ws[i] = w[i];
  for (int i = threadIdx.x; i < 16; i += blockDim.x) ws[16 * 27 + i] = bias[i];
  __syncthreads();
  const int Hh = Hp >> 1, Wh = Wp >> 1;
  const size_t total = (size_t)n * Hh * Wh;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(id % Wh);
    const size_t r = id / Wh;
    const int y = (int)(r % Hh);
    const int f = (int)(r / Hh);
    const float4* img = imgs + (size_t)f * Hp * Wp;
    float acc[16];
#pragma unroll
    for (int o = 0; o < 16; ++o) acc[o] = ws[16 * 27 + o];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int Y = 2 * y + ky - 1;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int X = 2 * x + kx - 1;
        if (Y >= 0 && Y < Hp && X >= 0 && X < Wp) {
          const float4 p = __ldg(img + (size_t)Y * Wp + X);
#pragma unroll
          for (int o = 0; o < 16; ++o) {  // weight [o][c][ky][kx]
            acc[o] = fmaf(p.x, ws[(o * 3 + 0) * 9 + ky * 3 + kx], acc[o]);
            acc[o] = fmaf(p.y, ws[(o * 3 + 1) * 9 + ky * 3 + kx], acc[o]);
            acc[o] = fmaf(p.z, ws[(o * 3 + 2) * 9 + ky * 3 + kx], acc[o]);
          }
        }
      }
    }
    float4* dst = reinterpret_cast<float4*>(e16 + id * 16);
#pragma unroll
    for (int q = 0; q < 4; ++q) dst[q] = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
  }
}

__global__ void encode_deconv_kernel(const float* __restrict__ e16, const float* __restrict__ w,
                                     const float* __restrict__ bias, uint2* __restrict__ feats, int n, int Hp,
                                     int Wp) {
  __shared__ float ws[16 * 4 * 16 + 4];  // ConvTranspose2d weight [16 in][4 out][4][4]
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) ws[i] = w[i];
  if (threadIdx.x < 4) ws[1024 + threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const int Hh = Hp >> 1, Wh = Wp >> 1;
  const size_t total = (size_t)n * Hp * Wp;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int X = (int)(id % Wp);
    const size_t r = id / Wp;
    const int Y = (int)(r % Hp);
    const int f = (int)(r / Hp);
    float o[4] = {ws[1024], ws[1025], ws[1026], ws[1027]};
    // out[2i-1+ky] += in[i]*w[ky]  ->  contributing input rows i = (Y+1)>>1 (ky = Y+1-2i in {0,1}) and i-1 (ky+2)
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      const int i = ((Y + 1) >> 1) - dy, ky = Y + 1 - 2 * i;
      if (i < 0 || i >= Hh) continue;
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const int j = ((X + 1) >> 1) - dx, kx = X + 1 - 2 * j;
        if (j < 0 || j >= Wh) continue;
        const float4* src = reinterpret_cast<const float4*>(e16 + (((size_t)f * Hh + i) * Wh + j) * 16);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 v = __ldg(src + q);
          const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int ci = 4 * q + c;
#pragma unroll
            for (int oc = 0; oc < 4; ++oc) o[oc] = fmaf(vv[c], ws[((ci * 4 + oc) * 4 + ky) * 4 + kx], o[oc]);
          }
        }
      }
    }
    // half4: the features only ever feed the 16-bit block inputs (the 4.7 fronts gather image and feature texels; 8 bytes
    // each instead of 16)
    feats[id] = make_uint2(Pack2<__half>::pack(o[0], o[1]), Pack2<__half>::pack(o[2], o[3]));
  }
}

// arch 4.7 block input: [w0.rgb, w1.rgb, warp(f0) (4), warp(f1) (4), t, mask, flow/s (4)] = 20 of 32 channels
// (block 0: [img0, img1, f0, f1, t] = 15), space-to-depth cell = 4 x 32 channels
template <typename T, int NLEV>
__global__ void front47_kernel(const uint2* __restrict__ imgs, const uint2* __restrict__ feats,
                               const FlowLevels lev, const BatchTasks tasks, int Hp, int Wp, int s,
                               T* __restrict__ x_s2d) {
  const int Hs = Hp / s, Ws = Wp / s;
  const size_t plane = (size_t)Hp * Wp;
  const float inv_s = 1.f / (float)s;
  {
    const int par = (int)(threadIdx.x & 1);
    const int xl = (int)(blockIdx.x * (blockDim.x >> 1) + (threadIdx.x >> 1));
    if (xl >= Ws) return;
    const int yl = (int)blockIdx.y * 2 + par;
    const int b = (int)blockIdx.z;
    const uint2* img0 = imgs + (size_t)tasks.f0[b] * plane;  // half4 planes: the block input is 16-bit anyway
    const uint2* img1 = imgs + (size_t)tasks.f1[b] * plane;
    const uint2* ft0 = feats + (size_t)tasks.f0[b] * plane;
    const uint2* ft1 = feats + (size_t)tasks.f1[b] * plane;
    const float t = tasks.t[b];
    const int ntap = (s == 1) ? 1 : 2;
    const int by = (s == 1) ? yl : s * yl + s / 2 - 1;
    const int bx = (s == 1) ? xl : s * xl + s / 2 - 1;
    float ch[20];
#pragma unroll
    for (int i = 0; i < 20; ++i) ch[i] = 0.f;
    float rowacc[2][20];
#pragma unroll
    for (int ty = 0; ty < 2; ++ty) {
      float colv[2][20];
#pragma unroll
      for (int tx = 0; tx < 2; ++tx) {
        if (ty < ntap && tx < ntap) {
          const int Y = by + ty, X = bx + tx;
          float* v = colv[tx];
          float4 a, c, fa, fc;
          if (NLEV == 0) {
            a = unpack_h4(__ldg(img0 + (size_t)Y * Wp + X));
            c = unpack_h4(__ldg(img1 + (size_t)Y * Wp + X));
            fa = unpack_h4(__ldg(ft0 + (size_t)Y * Wp + X));
            fc = unpack_h4(__ldg(ft1 + (size_t)Y * Wp + X));
            v[14] = t; v[15] = 0.f; v[16] = 0.f; v[17] = 0.f; v[18] = 0.f; v[19] = 0.f;
          } else {
            float4 f;
            float m;
            flow_at<(NLEV > 0 ? NLEV : 1)>(lev, b, Hp, Wp, Y, X, f, m);
            a = sample_border(img0, Hp, Wp, (float)X + f.x, (float)Y + f.y);
            c = sample_border(img1, Hp, Wp, (float)X + f.z, (float)Y + f.w);
            fa = sample_border4(ft0, Hp, Wp, (float)X + f.x, (float)Y + f.y);
            fc = sample_border4(ft1, Hp, Wp, (float)X + f.z, (float)Y + f.w);
            v[14] = t; v[15] = m; v[16] = f.x; v[17] = f.y; v[18] = f.z; v[19] = f.w;
          }
          v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = c.x; v[4] = c.y; v[5] = c.z;
          v[6] = fa.x; v[7] = fa.y; v[8] = fa.z; v[9] = fa.w; v[10] = fc.x; v[11] = fc.y; v[12] = fc.z; v[13] = fc.w;
        }
      }
#pragma unroll
      for (int i = 0; i < 20; ++i) rowacc[ty][i] = (ntap == 1) ? colv[0][i] : (colv[0][i] + colv[1][i]);
    }
#pragma unroll
    for (int i = 0; i < 20; ++i) ch[i] = (ntap == 1) ? rowacc[0][i] : 0.25f * (rowacc[0][i] + rowacc[1][i]);
#pragma unroll
    for (int i = 16; i < 20; ++i) ch[i] *= inv_s;
    const size_t cell = ((size_t)b * (Hs >> 1) + (yl >> 1)) * (Ws >> 1) + (xl >> 1);
    T* dst = x_s2d + cell * 128 + ((yl & 1) * 2 + (xl & 1)) * 32;
    uint4 q0, q1, q2;
    q0.x = Pack2<T>::pack(ch[0], ch[1]);   q0.y = Pack2<T>::pack(ch[2], ch[3]);
    q0.z = Pack2<T>::pack(ch[4], ch[5]);   q0.w = Pack2<T>::pack(ch[6], ch[7]);
    q1.x = Pack2<T>::pack(ch[8], ch[9]);   q1.y = Pack2<T>::pack(ch[10], ch[11]);
    q1.z = Pack2<T>::pack(ch[12], ch[13]); q1.w = Pack2<T>::pack(ch[14], ch[15]);
    q2.x = Pack2<T>::pack(ch[16], ch[17]); q2.y = Pack2<T>::pack(ch[18], ch[19]);
    q2.z = 0u; q2.w = 0u;
    reinterpret_cast<uint4*>(dst)[0] = q0;
    reinterpret_cast<uint4*>(dst)[1] = q1;
    reinterpret_cast<uint4*>(dst)[2] = q2;
    reinterpret_cast<uint4*>(dst)[3] = make_uint4(0u, 0u, 0u, 0u);
  }
}


// ---------------------------------------------------------------------------------------------
// arch 4.17 (rife417.pth): encode = Head_417 (rife_arch.py:356-375).  cnn0 (Conv2d 3->32, stride 2) + LeakyReLU runs
// here on the CUDA cores (0.45 GMAC per 1080p frame) and leaves a 16-bit NHWC [Hh][Wh][32] tensor for the tensor-core
// layers cnn1, cnn2 (32->32) and cnn3 (ConvTranspose 32->8, stored as the space-to-depth tensor [Hh][Wh][(a,b,oc)]).
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void head0_kernel(const float4* __restrict__ imgs, const float* __restrict__ w,
                             const float* __restrict__ bias, T* __restrict__ out, int n, int Hp, int Wp) {
  __shared__ float ws[32 * 27 + 32];
  for (int i = threadIdx.x; i < 32 * 27; i += blockDim.x) ws[i] = w[i];
  for (int i = threadIdx.x; i < 32; i += blockDim.x) ws[32 * 27 + i] = bias[i];
  __syncthreads();
  const int Hh = Hp >> 1, Wh = Wp >> 1;
  const int x = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (x >= Wh) return;
  const int y = (int)blockIdx.y, f = (int)blockIdx.z;
  const float4* img = imgs + (size_t)f * Hp * Wp;
  float acc[32];
#pragma unroll
  for (int o = 0; o < 32; ++o) acc[o] = ws[32 * 27 + o];
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int Y = 2 * y + ky - 1;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int X = 2 * x + kx - 1;
      if (Y >= 0 && Y < Hp && X >= 0 && X < Wp) {
        const float4 px = __ldg(img + (Y * Wp + X));
#pragma unroll
        for (int o = 0; o < 32; ++o) {  // weight [o][c][ky][kx]
          acc[o] = fmaf(px.x, ws[(o * 3 + 0) * 9 + ky * 3 + kx], acc[o]);
          acc[o] = fmaf(px.y, ws[(o * 3 + 1) * 9 + ky * 3 + kx], acc[o]);
          acc[o] = fmaf(px.z, ws[(o * 3 + 2) * 9 + ky * 3 + kx], acc[o]);
        }
      }
    }
  }
  uint4* dst = reinterpret_cast<uint4*>(out + (((size_t)f * Hh + y) * Wh + x) * 32);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float a0 = acc[8 * q + 2 * j], a1 = acc[8 * q + 2 * j + 1];
      o[j] = Pack2<T>::pack(fmaxf(a0, 0.2f * a0), fmaxf(a1, 0.2f * a1));
    }
    dst[q] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// 8-channel 16-bit features stored space-to-depth: pixel (Y, X) of frame plane `ft` ([Hh][Wh][4 x 8]) is one uint4
template <typename T>
__device__ __forceinline__ void load_feat8(const uint4* __restrict__ ft, int Wh, int Y, int X, float (&v)[8]) {
  const uint4 q = __ldg(ft + ((size_t)((Y >> 1) * Wh + (X >> 1)) * 4 + ((Y & 1) * 2 + (X & 1))));
  const float2 a = Pack2<T>::unpack(q.x), b = Pack2<T>::unpack(q.y), c = Pack2<T>::unpack(q.z), d = Pack2<T>::unpack(q.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}

// grid_sample(bilinear, border, align_corners=True) of the 8-channel feature plane at (sx, sy)
template <typename T>
__device__ __forceinline__ void sample_border8(const uint4* __restrict__ ft, int Hp, int Wp, float sx, float sy,
                                               float (&o)[8]) {
  sx = fminf(fmaxf(sx, 0.f), (float)(Wp - 1));
  sy = fminf(fmaxf(sy, 0.f), (float)(Hp - 1));
  const float fx0 = floorf(sx), fy0 = floorf(sy);
  const int x0 = (int)fx0, y0 = (int)fy0;
  const int x1 = min(x0 + 1, Wp - 1), y1 = min(y0 + 1, Hp - 1);
  const float ax = sx - fx0, ay = sy - fy0;
  const float w00 = (1.f - ax) * (1.f - ay), w01 = ax * (1.f - ay), w10 = (1.f - ax) * ay, w11 = ax * ay;
  float a[8], b[8], c[8], d[8];
  load_feat8<T>(ft, Wp >> 1, y0, x0, a);
  load_feat8<T>(ft, Wp >> 1, y0, x1, b);
  load_feat8<T>(ft, Wp >> 1, y1, x0, c);
  load_feat8<T>(ft, Wp >> 1, y1, x1, d);
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = a[i] * w00 + b[i] * w01 + c[i] * w10 + d[i] * w11;
}

// arch 4.17 block input: [w0.rgb, w1.rgb, warp(f0) (8), warp(f1) (8), t, mask, flow/s (4)] = 28 of 32 channels
// (block 0: [img0, img1, f0, f1, t] = 23), space-to-depth cell = 4 x 32 channels.  Same structure as front47_kernel;
// the 2x2 centre taps are summed row by row in the reference's order ((a + b) + (c + d)) * 0.25.
template <typename T, int NLEV>
__global__ void front417_kernel(const uint2* __restrict__ imgs, const uint4* __restrict__ feats,
                                const FlowLevels lev, const BatchTasks tasks, int Hp, int Wp, int s,
                                T* __restrict__ x_s2d) {
  const int Hs = Hp / s, Ws = Wp / s;
  const size_t plane = (size_t)Hp * Wp;
  const size_t fplane = plane / 4 * 4;  // uint4 per pixel: (Hp/2)*(Wp/2) cells x 4
  const float inv_s = 1.f / (float)s;
  const int par = (int)(threadIdx.x & 1);
  const int xl = (int)(blockIdx.x * (blockDim.x >> 1) + (threadIdx.x >> 1));
  if (xl >= Ws) return;
  const int yl = (int)blockIdx.y * 2 + par;
  const int b = (int)blockIdx.z;
  const uint2* img0 = imgs + (size_t)tasks.f0[b] * plane;  // half4 planes: the block input is 16-bit anyway
  const uint2* img1 = imgs + (size_t)tasks.f1[b] * plane;
  const uint4* ft0 = feats + (size_t)tasks.f0[b] * fplane;
  const uint4* ft1 = feats + (size_t)tasks.f1[b] * fplane;
  const float t = tasks.t[b];
  const int ntap = (s == 1) ? 1 : 2;
  const int by = (s == 1) ? yl : s * yl + s / 2 - 1;
  const int bx = (s == 1) ? xl : s * xl + s / 2 - 1;
  float ch[28];
#pragma unroll
  for (int ty = 0; ty < 2; ++ty) {
    float row[28];
#pragma unroll
    for (int tx = 0; tx < 2; ++tx) {
      if (ty < ntap && tx < ntap) {
        const int Y = by + ty, X = bx + tx;
        float v[28];
        float4 a, c;
        float fa[8], fc[8];
        if (NLEV == 0) {
          a = unpack_h4(__ldg(img0 + (size_t)Y * Wp + X));
          c = unpack_h4(__ldg(img1 + (size_t)Y * Wp + X));
          load_feat8<T>(ft0, Wp >> 1, Y, X, fa);
          load_feat8<T>(ft1, Wp >> 1, Y, X, fc);
          v[22] = t; v[23] = 0.f; v[24] = 0.f; v[25] = 0.f; v[26] = 0.f; v[27] = 0.f;
        } else {
          float4 f;
          float m;
          flow_at<(NLEV > 0 ? NLEV : 1)>(lev, b, Hp, Wp, Y, X, f, m);
          a = sample_border(img0, Hp, Wp, (float)X + f.x, (float)Y + f.y);
          c = sample_border(img1, Hp, Wp, (float)X + f.z, (float)Y + f.w);
          sample_border8<T>(ft0, Hp, Wp, (float)X + f.x, (float)Y + f.y, fa);
          sample_border8<T>(ft1, Hp, Wp, (float)X + f.z, (float)Y + f.w, fc);
          v[22] = t; v[23] = m; v[24] = f.x; v[25] = f.y; v[26] = f.z; v[27] = f.w;
        }
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = c.x; v[4] = c.y; v[5] = c.z;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          v[6 + i] = fa[i];
          v[14 + i] = fc[i];
        }
#pragma unroll
        for (int i = 0; i < 28; ++i) row[i] = (tx == 0) ? v[i] : row[i] + v[i];
      }
    }
    if (ty < ntap) {
#pragma unroll
      for (int i = 0; i < 28; ++i) ch[i] = (ty == 0) ? row[i] : ch[i] + row[i];
    }
  }
  if (ntap == 2) {
#pragma unroll
    for (int i = 0; i < 28; ++i) ch[i] *= 0.25f;
  }
#pragma unroll
  for (int i = 24; i < 28; ++i) ch[i] *= inv_s;  // flow is also divided by the scale (rife_arch.py:242-248)
  const size_t cell = ((size_t)b * (Hs >> 1) + (yl >> 1)) * (Ws >> 1) + (xl >> 1);
  T* dst = x_s2d + cell * 128 + ((yl & 1) * 2 + (xl & 1)) * 32;
  uint4 q[4];
  q[0] = make_uint4(Pack2<T>::pack(ch[0], ch[1]), Pack2<T>::pack(ch[2], ch[3]), Pack2<T>::pack(ch[4], ch[5]),
                    Pack2<T>::pack(ch[6], ch[7]));
  q[1] = make_uint4(Pack2<T>::pack(ch[8], ch[9]), Pack2<T>::pack(ch[10], ch[11]), Pack2<T>::pack(ch[12], ch[13]),
                    Pack2<T>::pack(ch[14], ch[15]));
  q[2] = make_uint4(Pack2<T>::pack(ch[16], ch[17]), Pack2<T>::pack(ch[18], ch[19]), Pack2<T>::pack(ch[20], ch[21]),
                    Pack2<T>::pack(ch[22], ch[23]));
  q[3] = make_uint4(Pack2<T>::pack(ch[24], ch[25]), Pack2<T>::pack(ch[26], ch[27]), 0u, 0u);
#pragma unroll
  for (int i = 0; i < 4; ++i) reinterpret_cast<uint4*>(dst)[i] = q[i];
}

// ---------------------------------------------------------------------------------------------
// arch 4.26 (rife426.pth): encode = Head (rife_arch.py:378-395; cnn0 on the CUDA cores via head0_kernel with the 16
// output channels zero-padded to 32, cnn1..cnn3 as tapconv layers) -> 4-channel 16-bit features stored space-to-depth
// ([Hh][Wh][4 x 4]: one uint2 per pixel).  Block input (rife_arch.py:521-526, :563-587):
//   block 0 : [img0, img1, f0 (4), f1 (4), t]                                                        = 15 of 32 channels
//   block i : [w0.rgb, w1.rgb, warp(f0), warp(f1), t, mask, feat (8), flow/s (4)]                     = 28 of 32 channels
// where `feat` = the previous block's 8 extra lastconv channels, bilinearly up-scaled to full resolution by its scale
// (rife_arch.py:267-274) and, like every other channel, down-scaled by 1/s here (2x2 centre taps).
// ---------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void load_feat4(const uint2* __restrict__ ft, int Wh, int Y, int X, float (&v)[4]) {
  const uint2 q = __ldg(ft + ((size_t)((Y >> 1) * Wh + (X >> 1)) * 4 + ((Y & 1) * 2 + (X & 1))));
  const float2 a = Pack2<T>::unpack(q.x), b = Pack2<T>::unpack(q.y);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}

template <typename T>
__device__ __forceinline__ void sample_border4h(const uint2* __restrict__ ft, int Hp, int Wp, float sx, float sy,
                                                float (&o)[4]) {
  sx = fminf(fmaxf(sx, 0.f), (float)(Wp - 1));
  sy = fminf(fmaxf(sy, 0.f), (float)(Hp - 1));
  const float fx0 = floorf(sx), fy0 = floorf(sy);
  const int x0 = (int)fx0, y0 = (int)fy0;
  const int x1 = min(x0 + 1, Wp - 1), y1 = min(y0 + 1, Hp - 1);
  const float ax = sx - fx0, ay = sy - fy0;
  const float w00 = (1.f - ax) * (1.f - ay), w01 = ax * (1.f - ay), w10 = (1.f - ax) * ay, w11 = ax * ay;
  float a[4], b[4], c[4], d[4];
  load_feat4<T>(ft, Wp >> 1, y0, x0, a);
  load_feat4<T>(ft, Wp >> 1, y0, x1, b);
  load_feat4<T>(ft, Wp >> 1, y1, x0, c);
  load_feat4<T>(ft, Wp >> 1, y1, x1, d);
#pragma unroll
  for (int i = 0; i < 4; ++i) o[i] = a[i] * w00 + b[i] * w01 + c[i] * w10 + d[i] * w11;
}

template <typename T>
__device__ __forceinline__ void unpack8(const uint4 q, float (&v)[8]) {
  const float2 a = Pack2<T>::unpack(q.x), b = Pack2<T>::unpack(q.y), c = Pack2<T>::unpack(q.z), d = Pack2<T>::unpack(q.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}

// F.interpolate(scale_factor=s, bilinear, align_corners=False) of the 8-channel plane pf [Hs][Ws] at full-res (Y, X)
template <typename T>
__device__ __forceinline__ void up_feat8(const uint4* __restrict__ pf, int Hs, int Ws, int s, float inv_s, int Y, int X,
                                         float (&o)[8]) {
  if (s == 1) {
    unpack8<T>(__ldg(pf + (Y * Ws + X)), o);
    return;
  }
  const float sy = fmaxf(((float)Y + 0.5f) * inv_s - 0.5f, 0.f);
  const float sx = fmaxf(((float)X + 0.5f) * inv_s - 0.5f, 0.f);
  const int y0 = min((int)sy, Hs - 1), x0 = min((int)sx, Ws - 1);
  const int dx = (x0 + 1 < Ws) ? 1 : 0, dyw = (y0 + 1 < Hs) ? Ws : 0;
  const float ly = sy - (float)y0, lx = sx - (float)x0;
  const float hy = 1.f - ly, hx = 1.f - lx;
  const int o00 = y0 * Ws + x0;
  float a[8], b[8], c[8], d[8];
  unpack8<T>(__ldg(pf + o00), a);
  unpack8<T>(__ldg(pf + o00 + dx), b);
  unpack8<T>(__ldg(pf + o00 + dyw), c);
  unpack8<T>(__ldg(pf + o00 + dyw + dx), d);
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = hy * (hx * a[i] + lx * b[i]) + ly * (hx * c[i] + lx * d[i]);
}

template <typename T, int NLEV>
__global__ void front426_kernel(const uint2* __restrict__ imgs, const uint2* __restrict__ feats,
                                const uint4* __restrict__ prev_feat, int prev_s, const FlowLevels lev,
                                const BatchTasks tasks, int Hp, int Wp, int s, T* __restrict__ x_s2d) {
  const int Hs = Hp / s, Ws = Wp / s;
  const size_t plane = (size_t)Hp * Wp;
  const float inv_s = 1.f / (float)s;
  const int par = (int)(threadIdx.x & 1);
  const int xl = (int)(blockIdx.x * (blockDim.x >> 1) + (threadIdx.x >> 1));
  if (xl >= Ws) return;
  const int yl = (int)blockIdx.y * 2 + par;
  const int b = (int)blockIdx.z;
  const uint2* img0 = imgs + (size_t)tasks.f0[b] * plane;
  const uint2* img1 = imgs + (size_t)tasks.f1[b] * plane;
  const uint2* ft0 = feats + (size_t)tasks.f0[b] * plane;  // one uint2 per pixel
  const uint2* ft1 = feats + (size_t)tasks.f1[b] * plane;
  const int pHs = NLEV ? Hp / prev_s : 1, pWs = NLEV ? Wp / prev_s : 1;
  const uint4* pf = NLEV ? prev_feat + (size_t)b * pHs * pWs : nullptr;
  const float pinv = NLEV ? 1.f / (float)prev_s : 1.f;
  const float t = tasks.t[b];
  const int ntap = (s == 1) ? 1 : 2;
  const int by = (s == 1) ? yl : s * yl + s / 2 - 1;
  const int bx = (s == 1) ? xl : s * xl + s / 2 - 1;
  float ch[28];
#pragma unroll
  for (int ty = 0; ty < 2; ++ty) {
    float row[28];
#pragma unroll
    for (int tx = 0; tx < 2; ++tx) {
      if (ty < ntap && tx < ntap) {
        const int Y = by + ty, X = bx + tx;
        float v[28];
        float4 a, c;
        float fa[4], fc[4];
        if (NLEV == 0) {
          a = unpack_h4(__ldg(img0 + (size_t)Y * Wp + X));
          c = unpack_h4(__ldg(img1 + (size_t)Y * Wp + X));
          load_feat4<T>(ft0, Wp >> 1, Y, X, fa);
          load_feat4<T>(ft1, Wp >> 1, Y, X, fc);
          v[14] = t;
#pragma unroll
          for (int i = 15; i < 28; ++i) v[i] = 0.f;
        } else {
          float4 f;
          float m;
          flow_at<(NLEV > 0 ? NLEV : 1)>(lev, b, Hp, Wp, Y, X, f, m);
          a = sample_border(img0, Hp, Wp, (float)X + f.x, (float)Y + f.y);
          c = sample_border(img1, Hp, Wp, (float)X + f.z, (float)Y + f.w);
          sample_border4h<T>(ft0, Hp, Wp, (float)X + f.x, (float)Y + f.y, fa);
          sample_border4h<T>(ft1, Hp, Wp, (float)X + f.z, (float)Y + f.w, fc);
          float pe[8];
          up_feat8<T>(pf, pHs, pWs, prev_s, pinv, Y, X, pe);
          v[14] = t; v[15] = m;
#pragma unroll
          for (int i = 0; i < 8; ++i) v[16 + i] = pe[i];
          v[24] = f.x; v[25] = f.y; v[26] = f.z; v[27] = f.w;
        }
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = c.x; v[4] = c.y; v[5] = c.z;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          v[6 + i] = fa[i];
          v[10 + i] = fc[i];
        }
#pragma unroll
        for (int i = 0; i < 28; ++i) row[i] = (tx == 0) ? v[i] : row[i] + v[i];
      }
    }
    if (ty < ntap) {
#pragma unroll
      for (int i = 0; i < 28; ++i) ch[i] = (ty == 0) ? row[i] : ch[i] + row[i];
    }
  }
  if (ntap == 2) {
#pragma unroll
    for (int i = 0; i < 28; ++i) ch[i] *= 0.25f;
  }
#pragma unroll
  for (int i = 24; i < 28; ++i) ch[i] *= inv_s;  // flow is also divided by the scale (rife_arch.py:242-248)
  const size_t cell = ((size_t)b * (Hs >> 1) + (yl >> 1)) * (Ws >> 1) + (xl >> 1);
  T* dst = x_s2d + cell * 128 + ((yl & 1) * 2 + (xl & 1)) * 32;
  uint4 q[4];
  q[0] = make_uint4(Pack2<T>::pack(ch[0], ch[1]), Pack2<T>::pack(ch[2], ch[3]), Pack2<T>::pack(ch[4], ch[5]),
                    Pack2<T>::pack(ch[6], ch[7]));
  q[1] = make_uint4(Pack2<T>::pack(ch[8], ch[9]), Pack2<T>::pack(ch[10], ch[11]), Pack2<T>::pack(ch[12], ch[13]),
                    Pack2<T>::pack(ch[14], ch[15]));
  q[2] = make_uint4(Pack2<T>::pack(ch[16], ch[17]), Pack2<T>::pack(ch[18], ch[19]), Pack2<T>::pack(ch[20], ch[21]),
                    Pack2<T>::pack(ch[22], ch[23]));
  q[3] = make_uint4(Pack2<T>::pack(ch[24], ch[25]), Pack2<T>::pack(ch[26], ch[27]), 0u, 0u);
#pragma unroll
  for (int i = 0; i < 4; ++i) reinterpret_cast<uint4*>(dst)[i] = q[i];
}

// debug / tests only: materialise the accumulated full-resolution flow and mask

// ---- up-scaled blocks (node scale_factor 2 / 4: block scale 1/k, k = 2 or 4) - arch 4.6 ------------------------------
// The reference interpolates the full-resolution block input UP by k before conv0 (rife_arch.py:238-249 with
// scale < 1): x = interpolate(cat(warped img0, warped img1, t, mask), k), flow = interpolate(flow, k) * k, bilinear,
// align_corners=False.  One thread = one cell of the k-times finer grid: source position (cell + 0.5) / k - 0.5 clamped at
// 0, the four surrounding full-resolution pixels each evaluated like front_kernel does (dense flow / mask planes F, M -
// every earlier level has been folded into them - and the two border-clamped warps), then mixed.  Same 16-channel
// space-to-depth store as front_kernel.
template <typename T>
__global__ void front_up_kernel(const uint2* __restrict__ imgs, const float4* __restrict__ F, const float* __restrict__ M,
                                const BatchTasks tasks, int Hp, int Wp, int k, T* __restrict__ x_s2d) {
  const int Hs = Hp * k, Ws = Wp * k;
  const size_t plane = (size_t)Hp * Wp;
  const float inv_k = 1.f / (float)k;
  const int par = (int)(threadIdx.x & 1);
  const int xl = (int)(blockIdx.x * (blockDim.x >> 1) + (threadIdx.x >> 1));
  if (xl >= Ws) return;
  const int yl = (int)blockIdx.y * 2 + par;
  const int b = (int)blockIdx.z;
  const uint2* img0 = imgs + (size_t)tasks.f0[b] * plane;
  const uint2* img1 = imgs + (size_t)tasks.f1[b] * plane;
  const float t = tasks.t[b];
  const float sy = fmaxf(((float)yl + 0.5f) * inv_k - 0.5f, 0.f), sx = fmaxf(((float)xl + 0.5f) * inv_k - 0.5f, 0.f);
  const int y0 = min((int)sy, Hp - 1), x0 = min((int)sx, Wp - 1);
  const int y1 = min(y0 + 1, Hp - 1), x1 = min(x0 + 1, Wp - 1);
  const float ly = sy - (float)y0, lx = sx - (float)x0;
  const float wq[4] = {(1.f - ly) * (1.f - lx), (1.f - ly) * lx, ly * (1.f - lx), ly * lx};
  const int qy[4] = {y0, y0, y1, y1}, qx[4] = {x0, x1, x0, x1};
  float ch[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) ch[i] = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int Y = qy[q], X = qx[q];
    const size_t pid = ((size_t)b * Hp + Y) * Wp + X;
    const float4 f = F[pid];
    const float m = M[pid];
    const float4 a = sample_border(img0, Hp, Wp, (float)X + f.x, (float)Y + f.y);
    const float4 c = sample_border(img1, Hp, Wp, (float)X + f.z, (float)Y + f.w);
    const float v[12] = {a.x, a.y, a.z, c.x, c.y, c.z, t, m, f.x, f.y, f.z, f.w};
#pragma unroll
    for (int i = 0; i < 12; ++i) ch[i] = fmaf(v[i], wq[q], ch[i]);
  }
#pragma unroll
  for (int i = 8; i < 12; ++i) ch[i] *= (float)k;  // flow * (1 / scale), rife_arch.py:245-248
  const size_t cell = ((size_t)b * (Hs >> 1) + (yl >> 1)) * (Ws >> 1) + (xl >> 1);
  T* dst = x_s2d + cell * 64 + ((yl & 1) * 2 + (xl & 1)) * 16;
  uint4 lo, hi;
  lo.x = Pack2<T>::pack(ch[0], ch[1]);
  lo.y = Pack2<T>::pack(ch[2], ch[3]);
  lo.z = Pack2<T>::pack(ch[4], ch[5]);
  lo.w = Pack2<T>::pack(ch[6], ch[7]);
  hi.x = Pack2<T>::pack(ch[8], ch[9]);
  hi.y = Pack2<T>::pack(ch[10], ch[11]);
  hi.z = 0u;
  hi.w = 0u;
  reinterpret_cast<uint4*>(dst)[0] = lo;
  reinterpret_cast<uint4*>(dst)[1] = hi;
}

// arch 4.7 variant: the 32-channel layout of front47_kernel ([w0.rgb, w1.rgb, warp(f0) 4, warp(f1) 4, t, mask, flow 4])
template <typename T>
__global__ void front_up47_kernel(const uint2* __restrict__ imgs, const uint2* __restrict__ feats, const float4* __restrict__ F,
                                  const float* __restrict__ M, const BatchTasks tasks, int Hp, int Wp, int k,
                                  T* __restrict__ x_s2d) {
  const int Hs = Hp * k, Ws = Wp * k;
  const size_t plane = (size_t)Hp * Wp;
  const float inv_k = 1.f / (float)k;
  const int par = (int)(threadIdx.x & 1);
  const int xl = (int)(blockIdx.x * (blockDim.x >> 1) + (threadIdx.x >> 1));
  if (xl >= Ws) return;
  const int yl = (int)blockIdx.y * 2 + par;
  const int b = (int)blockIdx.z;
  const uint2* img0 = imgs + (size_t)tasks.f0[b] * plane;
  const uint2* img1 = imgs + (size_t)tasks.f1[b] * plane;
  const uint2* ft0 = feats + (size_t)tasks.f0[b] * plane;
  const uint2* ft1 = feats + (size_t)tasks.f1[b] * plane;
  const float t = tasks.t[b];
  const float sy = fmaxf(((float)yl + 0.5f) * inv_k - 0.5f, 0.f), sx = fmaxf(((float)xl + 0.5f) * inv_k - 0.5f, 0.f);
  const int y0 = min((int)sy, Hp - 1), x0 = min((int)sx, Wp - 1);
  const int y1 = min(y0 + 1, Hp - 1), x1 = min(x0 + 1, Wp - 1);
  const float ly = sy - (float)y0, lx = sx - (float)x0;
  const float wq[4] = {(1.f - ly) * (1.f - lx), (1.f - ly) * lx, ly * (1.f - lx), ly * lx};
  const int qy[4] = {y0, y0, y1, y1}, qx[4] = {x0, x1, x0, x1};
  float ch[20];
#pragma unroll
  for (int i = 0; i < 20; ++i) ch[i] = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int Y = qy[q], X = qx[q];
    const size_t pid = ((size_t)b * Hp + Y) * Wp + X;
    const float4 f = F[pid];
    const float m = M[pid];
    const float4 a = sample_border(img0, Hp, Wp, (float)X + f.x, (float)Y + f.y);
    const float4 c = sample_border(img1, Hp, Wp, (float)X + f.z, (float)Y + f.w);
    const float4 fa = sample_border4(ft0, Hp, Wp, (float)X + f.x, (float)Y + f.y);
    const float4 fc = sample_border4(ft1, Hp, Wp, (float)X + f.z, (float)Y + f.w);
    const float v[20] = {a.x, a.y, a.z, c.x, c.y, c.z, fa.x, fa.y, fa.z, fa.w, fc.x, fc.y, fc.z, fc.w, t, m, f.x, f.y, f.z, f.w};
#pragma unroll
    for (int i = 0; i < 20; ++i) ch[i] = fmaf(v[i], wq[q], ch[i]);
  }
#pragma unroll
  for (int i = 16; i < 20; ++i) ch[i] *= (float)k;
  const size_t cell = ((size_t)b * (Hs >> 1) + (yl >> 1)) * (Ws >> 1) + (xl >> 1);
  T* dst = x_s2d + cell * 128 + ((yl & 1) * 2 + (xl & 1)) * 32;
  uint4 q0, q1, q2;
  q0.x = Pack2<T>::pack(ch[0], ch[1]);   q0.y = Pack2<T>::pack(ch[2], ch[3]);
  q0.z = Pack2<T>::pack(ch[4], ch[5]);   q0.w = Pack2<T>::pack(ch[6], ch[7]);
  q1.x = Pack2<T>::pack(ch[8], ch[9]);   q1.y = Pack2<T>::pack(ch[10], ch[11]);
  q1.z = Pack2<T>::pack(ch[12], ch[13]); q1.w = Pack2<T>::pack(ch[14], ch[15]);
  q2.x = Pack2<T>::pack(ch[16], ch[17]); q2.y = Pack2<T>::pack(ch[18], ch[19]);
  q2.z = 0u; q2.w = 0u;
  reinterpret_cast<uint4*>(dst)[0] = q0;
  reinterpret_cast<uint4*>(dst)[1] = q1;
  reinterpret_cast<uint4*>(dst)[2] = q2;
  reinterpret_cast<uint4*>(dst)[3] = make_uint4(0u, 0u, 0u, 0u);
}

// arch 4.17 variant: the 32-channel layout of front417_kernel ([w0.rgb, w1.rgb, warp(f0) 8, warp(f1) 8, t, mask, flow 4])
template <typename T>
__global__ void front_up417_kernel(const uint2* __restrict__ imgs, const uint4* __restrict__ feats, const float4* __restrict__ F,
                                   const float* __restrict__ M, const BatchTasks tasks, int Hp, int Wp, int k,
                                   T* __restrict__ x_s2d) {
  const int Hs = Hp * k, Ws = Wp * k;
  const size_t plane = (size_t)Hp * Wp;
  const size_t fplane = plane / 4 * 4;
  const float inv_k = 1.f / (float)k;
  const int par = (int)(threadIdx.x & 1);
  const int xl = (int)(blockIdx.x * (blockDim.x >> 1) + (threadIdx.x >> 1));
  if (xl >= Ws) return;
  const int yl = (int)blockIdx.y * 2 + par;
  const int b = (int)blockIdx.z;
  const uint2* img0 = imgs + (size_t)tasks.f0[b] * plane;
  const uint2* img1 = imgs + (size_t)tasks.f1[b] * plane;
  const uint4* ft0 = feats + (size_t)tasks.f0[b] * fplane;
  const uint4* ft1 = feats + (size_t)tasks.f1[b] * fplane;
  const float t = tasks.t[b];
  const float sy = fmaxf(((float)yl + 0.5f) * inv_k - 0.5f, 0.f), sx = fmaxf(((float)xl + 0.5f) * inv_k - 0.5f, 0.f);
  const int y0 = min((int)sy, Hp - 1), x0 = min((int)sx, Wp - 1);
  const int y1 = min(y0 + 1, Hp - 1), x1 = min(x0 + 1, Wp - 1);
  const float ly = sy - (float)y0, lx = sx - (float)x0;
  const float wq[4] = {(1.f - ly) * (1.f - lx), (1.f - ly) * lx, ly * (1.f - lx), ly * lx};
  const int qy[4] = {y0, y0, y1, y1}, qx[4] = {x0, x1, x0, x1};
  float ch[28];
#pragma unroll
  for (int i = 0; i < 28; ++i) ch[i] = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int Y = qy[q], X = qx[q];
    const size_t pid = ((size_t)b * Hp + Y) * Wp + X;
    const float4 f = F[pid];
    const float m = M[pid];
    const float4 a = sample_border(img0, Hp, Wp, (float)X + f.x, (float)Y + f.y);
    const float4 c = sample_border(img1, Hp, Wp, (float)X + f.z, (float)Y + f.w);
    float fa[8], fc[8];
    sample_border8<T>(ft0, Hp, Wp, (float)X + f.x, (float)Y + f.y, fa);
    sample_border8<T>(ft1, Hp, Wp, (float)X + f.z, (float)Y + f.w, fc);
    float v[28] = {a.x, a.y, a.z, c.x, c.y, c.z};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      v[6 + i] = fa[i];
      v[14 + i] = fc[i];
    }
    v[22] = t; v[23] = m; v[24] = f.x; v[25] = f.y; v[26] = f.z; v[27] = f.w;
#pragma unroll
    for (int i = 0; i < 28; ++i) ch[i] = fmaf(v[i], wq[q], ch[i]);
  }
#pragma unroll
  for (int i = 24; i < 28; ++i) ch[i] *= (float)k;
  const size_t cell = ((size_t)b * (Hs >> 1) + (yl >> 1)) * (Ws >> 1) + (xl >> 1);
  T* dst = x_s2d + cell * 128 + ((yl & 1) * 2 + (xl & 1)) * 32;
  uint4 q4[4];
  q4[0] = make_uint4(Pack2<T>::pack(ch[0], ch[1]), Pack2<T>::pack(ch[2], ch[3]), Pack2<T>::pack(ch[4], ch[5]),
                     Pack2<T>::pack(ch[6], ch[7]));
  q4[1] = make_uint4(Pack2<T>::pack(ch[8], ch[9]), Pack2<T>::pack(ch[10], ch[11]), Pack2<T>::pack(ch[12], ch[13]),
                     Pack2<T>::pack(ch[14], ch[15]));
  q4[2] = make_uint4(Pack2<T>::pack(ch[16], ch[17]), Pack2<T>::pack(ch[18], ch[19]), Pack2<T>::pack(ch[20], ch[21]),
                     Pack2<T>::pack(ch[22], ch[23]));
  q4[3] = make_uint4(Pack2<T>::pack(ch[24], ch[25]), Pack2<T>::pack(ch[26], ch[27]), 0u, 0u);
#pragma unroll
  for (int i = 0; i < 4; ++i) reinterpret_cast<uint4*>(dst)[i] = q4[i];
}

// interpolate(scale_factor = 1 / k) of an 8-channel plane pf [k Hp][k Wp] at full-res (Y, X): the two central taps per axis
template <typename T>
__device__ __forceinline__ void down_feat8(const uint4* __restrict__ pf, int Ws, int k, int Y, int X, float (&o)[8]) {
  const size_t base = (size_t)(k * Y + k / 2 - 1) * Ws + (size_t)(k * X + k / 2 - 1);
  float a[8], b[8], c[8], d[8];
  unpack8<T>(__ldg(pf + base), a);
  unpack8<T>(__ldg(pf + base + 1), b);
  unpack8<T>(__ldg(pf + base + Ws), c);
  unpack8<T>(__ldg(pf + base + Ws + 1), d);
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = 0.5f * (0.5f * a[i] + 0.5f * b[i]) + 0.5f * (0.5f * c[i] + 0.5f * d[i]);
}

// arch 4.26 variant: the layout of front426_kernel ([w0.rgb, w1.rgb, warp(f0) 4, warp(f1) 4, t, mask, feat 8, flow 4]); `feat`
// = the previous block's 8 extra lastconv channels brought to full resolution (up by its scale prev_s, or - when that block
// was itself up-scaled by prev_k - down by prev_k; rife_arch.py:267-274), then up-scaled with everything else.
template <typename T>
__global__ void front_up426_kernel(const uint2* __restrict__ imgs, const uint2* __restrict__ feats,
                                   const uint4* __restrict__ prev_feat, int prev_s, int prev_k, const float4* __restrict__ F,
                                   const float* __restrict__ M, const BatchTasks tasks, int Hp, int Wp, int k,
                                   T* __restrict__ x_s2d) {
  const int Hs = Hp * k, Ws = Wp * k;
  const size_t plane = (size_t)Hp * Wp;
  const size_t fplane = plane / 4 * 4;
  const float inv_k = 1.f / (float)k;
  const int par = (int)(threadIdx.x & 1);
  const int xl = (int)(blockIdx.x * (blockDim.x >> 1) + (threadIdx.x >> 1));
  if (xl >= Ws) return;
  const int yl = (int)blockIdx.y * 2 + par;
  const int b = (int)blockIdx.z;
  const uint2* img0 = imgs + (size_t)tasks.f0[b] * plane;
  const uint2* img1 = imgs + (size_t)tasks.f1[b] * plane;
  const uint2* ft0 = feats + (size_t)tasks.f0[b] * fplane;
  const uint2* ft1 = feats + (size_t)tasks.f1[b] * fplane;
  const int pHs = prev_k > 1 ? Hp * prev_k : Hp / prev_s, pWs = prev_k > 1 ? Wp * prev_k : Wp / prev_s;
  const uint4* pf = prev_feat + (size_t)b * pHs * pWs;
  const float pinv = 1.f / (float)prev_s;
  const float t = tasks.t[b];
  const float sy = fmaxf(((float)yl + 0.5f) * inv_k - 0.5f, 0.f), sx = fmaxf(((float)xl + 0.5f) * inv_k - 0.5f, 0.f);
  const int y0 = min((int)sy, Hp - 1), x0 = min((int)sx, Wp - 1);
  const int y1 = min(y0 + 1, Hp - 1), x1 = min(x0 + 1, Wp - 1);
  const float ly = sy - (float)y0, lx = sx - (float)x0;
  const float wq[4] = {(1.f - ly) * (1.f - lx), (1.f - ly) * lx, ly * (1.f - lx), ly * lx};
  const int qy[4] = {y0, y0, y1, y1}, qx[4] = {x0, x1, x0, x1};
  float ch[28];
#pragma unroll
  for (int i = 0; i < 28; ++i) ch[i] = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int Y = qy[q], X = qx[q];
    const size_t pid = ((size_t)b * Hp + Y) * Wp + X;
    const float4 f = F[pid];
    const float m = M[pid];
    const float4 a = sample_border(img0, Hp, Wp, (float)X + f.x, (float)Y + f.y);
    const float4 c = sample_border(img1, Hp, Wp, (float)X + f.z, (float)Y + f.w);
    float fa[4], fc[4], pe[8];
    sample_border4h<T>(ft0, Hp, Wp, (float)X + f.x, (float)Y + f.y, fa);
    sample_border4h<T>(ft1, Hp, Wp, (float)X + f.z, (float)Y + f.w, fc);
    if (prev_k > 1)
      down_feat8<T>(pf, pWs, prev_k, Y, X, pe);
    else
      up_feat8<T>(pf, pHs, pWs, prev_s, pinv, Y, X, pe);
    float v[28] = {a.x, a.y, a.z, c.x, c.y, c.z, fa[0], fa[1], fa[2], fa[3], fc[0], fc[1], fc[2], fc[3], t, m};
#pragma unroll
    for (int i = 0; i < 8; ++i) v[16 + i] = pe[i];
    v[24] = f.x; v[25] = f.y; v[26] = f.z; v[27] = f.w;
#pragma unroll
    for (int i = 0; i < 28; ++i) ch[i] = fmaf(v[i], wq[q], ch[i]);
  }
#pragma unroll
  for (int i = 24; i < 28; ++i) ch[i] *= (float)k;
  const size_t cell = ((size_t)b * (Hs >> 1) + (yl >> 1)) * (Ws >> 1) + (xl >> 1);
  T* dst = x_s2d + cell * 128 + ((yl & 1) * 2 + (xl & 1)) * 32;
  uint4 q4[4];
  q4[0] = make_uint4(Pack2<T>::pack(ch[0], ch[1]), Pack2<T>::pack(ch[2], ch[3]), Pack2<T>::pack(ch[4], ch[5]),
                     Pack2<T>::pack(ch[6], ch[7]));
  q4[1] = make_uint4(Pack2<T>::pack(ch[8], ch[9]), Pack2<T>::pack(ch[10], ch[11]), Pack2<T>::pack(ch[12], ch[13]),
                     Pack2<T>::pack(ch[14], ch[15]));
  q4[2] = make_uint4(Pack2<T>::pack(ch[16], ch[17]), Pack2<T>::pack(ch[18], ch[19]), Pack2<T>::pack(ch[20], ch[21]),
                     Pack2<T>::pack(ch[22], ch[23]));
  q4[3] = make_uint4(Pack2<T>::pack(ch[24], ch[25]), Pack2<T>::pack(ch[26], ch[27]), 0u, 0u);
#pragma unroll
  for (int i = 0; i < 4; ++i) reinterpret_cast<uint4*>(dst)[i] = q4[i];
}

// The block's output T (flow increments float4 + mask, k times finer than full resolution) back onto the dense planes:
// interpolate(T, scale_factor = 1 / k) takes the two central taps k p + k/2 - 1, k p + k/2 per axis with weight 1/2 (for
// k = 2 the 2x2 mean), flow is multiplied by the scale 1 / k (rife_arch.py:263-266) and added; the mask is added (arch 4.6) or
// replaces the old one (arch 4.7+, rife_arch.py:698-699).
__global__ void fold_down_kernel(const float4* __restrict__ tf, const float* __restrict__ tm, int k, float4* __restrict__ F,
                                 float* __restrict__ M, int B, int Hp, int Wp, int mask_replace) {
  const size_t total = (size_t)B * Hp * Wp;
  const int Ws = Wp * k;
  const float inv_k = 1.f / (float)k;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int X = (int)(id % Wp);
    const int Y = (int)((id / Wp) % Hp);
    const int b = (int)(id / ((size_t)Wp * Hp));
    const size_t base = ((size_t)b * Hp * k + (size_t)(k * Y + k / 2 - 1)) * Ws + (size_t)(k * X + k / 2 - 1);
    const float4 a = tf[base], c = tf[base + 1], d = tf[base + Ws], e = tf[base + Ws + 1];
    const float ma = tm[base], mc = tm[base + 1], md = tm[base + Ws], me = tm[base + Ws + 1];
    float4 f = F[id];
    f.x += (0.5f * (0.5f * a.x + 0.5f * c.x) + 0.5f * (0.5f * d.x + 0.5f * e.x)) * inv_k;
    f.y += (0.5f * (0.5f * a.y + 0.5f * c.y) + 0.5f * (0.5f * d.y + 0.5f * e.y)) * inv_k;
    f.z += (0.5f * (0.5f * a.z + 0.5f * c.z) + 0.5f * (0.5f * d.z + 0.5f * e.z)) * inv_k;
    f.w += (0.5f * (0.5f * a.w + 0.5f * c.w) + 0.5f * (0.5f * d.w + 0.5f * e.w)) * inv_k;
    F[id] = f;
    const float md_ = 0.5f * (0.5f * ma + 0.5f * mc) + 0.5f * (0.5f * md + 0.5f * me);
    M[id] = mask_replace ? md_ : M[id] + md_;
  }
}

template <int NLEV>
__global__ void materialize_kernel(const FlowLevels lev, float4* __restrict__ flow, float* __restrict__ mask, int B,
                                   int Hp, int Wp) {
  const size_t total = (size_t)B * Hp * Wp;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(id % Wp);
    const size_t r = id / Wp;
    float4 f;
    float m;
    flow_at<NLEV>(lev, (int)(r / Hp), Hp, Wp, (int)(r % Hp), x, f, m);
    flow[id] = f;
    mask[id] = m;
  }
}

template <int NLEV>
__global__ void final_kernel(const float4* __restrict__ imgs, const FlowLevels lev, const BatchTasks tasks, int Hp,
                             int Wp, int H, int W, float* __restrict__ out) {
  const size_t plane = (size_t)Hp * Wp;
  {
    const int x = (int)(blockIdx.x * blockDim.x + threadIdx.x);
    if (x >= W) return;
    const int y = (int)blockIdx.y;
    const int b = (int)blockIdx.z;
    const size_t id = ((size_t)b * H + y) * W + x;
    float4 f;
    float m;
    flow_at<NLEV>(lev, b, Hp, Wp, y, x, f, m);
    const float4 a = sample_border(imgs + (size_t)tasks.f0[b] * plane, Hp, Wp, (float)x + f.x, (float)y + f.y);
    const float4 c = sample_border(imgs + (size_t)tasks.f1[b] * plane, Hp, Wp, (float)x + f.z, (float)y + f.w);
    const float sg = 1.f / (1.f + expf(-m));
    float* o = out + id * 3;
    o[0] = clamp01(a.x * sg + c.x * (1.f - sg));
    o[1] = clamp01(a.y * sg + c.y * (1.f - sg));
    o[2] = clamp01(a.z * sg + c.z * (1.f - sg));
  }
}

// stand-alone warp, NHWC fp32 with C channels (C % 4 == 0 uses 128-bit loads): img [B,H,W,C], flow [B,H,W,2]
template <int VEC>
__global__ void warp_kernel(const float* __restrict__ img, const float* __restrict__ flow, float* __restrict__ out,
                            int B, int H, int W, int C) {
  const int cv = C / VEC;  // vectors per pixel
  const size_t total = (size_t)B * H * W * cv;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int v = (int)(id % cv);
    const size_t pix = id / cv;
    const int x = (int)(pix % W);
    const size_t r = pix / W;
    const int y = (int)(r % H);
    const int b = (int)(r / H);
    const float2 f = __ldg(reinterpret_cast<const float2*>(flow) + pix);
    const float sx = fminf(fmaxf((float)x + f.x, 0.f), (float)(W - 1));
    const float sy = fminf(fmaxf((float)y + f.y, 0.f), (float)(H - 1));
    const float fx0 = floorf(sx), fy0 = floorf(sy);
    const int x0 = (int)fx0, y0 = (int)fy0;
    const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
    const float ax = sx - fx0, ay = sy - fy0;
    const float w00 = (1.f - ax) * (1.f - ay), w01 = ax * (1.f - ay), w10 = (1.f - ax) * ay, w11 = ax * ay;
    const float* base = img + (size_t)b * H * W * C + (size_t)v * VEC;
    const float* p00 = base + ((size_t)y0 * W + x0) * C;
    const float* p01 = base + ((size_t)y0 * W + x1) * C;
    const float* p10 = base + ((size_t)y1 * W + x0) * C;
    const float* p11 = base + ((size_t)y1 * W + x1) * C;
    float* o = out + pix * C + (size_t)v * VEC;
    if (VEC == 4) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(p00));
      const float4 bq = __ldg(reinterpret_cast<const float4*>(p01));
      const float4 c = __ldg(reinterpret_cast<const float4*>(p10));
      const float4 d = __ldg(reinterpret_cast<const float4*>(p11));
      float4 q;
      q.x = a.x * w00 + bq.x * w01 + c.x * w10 + d.x * w11;
      q.y = a.y * w00 + bq.y * w01 + c.y * w10 + d.y * w11;
      q.z = a.z * w00 + bq.z * w01 + c.z * w10 + d.z * w11;
      q.w = a.w * w00 + bq.w * w01 + c.w * w10 + d.w * w11;
      *reinterpret_cast<float4*>(o) = q;
    } else {
      o[0] = __ldg(p00) * w00 + __ldg(p01) * w01 + __ldg(p10) * w10 + __ldg(p11) * w11;
    }
  }
}

inline int grid_for(size_t total, int block) {
  size_t g = (total + block - 1) / block;
  const size_t cap = 132 * 32;  // grid-stride loops: a few waves of the 132 SMs
  return (int)(g < cap ? (g ? g : 1) : cap);
}

}  // namespace

cudaError_t launch_prep_frames(const float* frames, int n, int H, int W, int cstride, float4* imgs, uint2* imgs_h,
                               int Hp, int Wp, cudaStream_t st) {
  const size_t total = (size_t)n * Hp * Wp;
  VFI_LAUNCH((prep_frames_kernel), grid_for(total, 256), 256, 0, st, frames, n, H, W, cstride, imgs, imgs_h, Hp, Wp);
  return cudaGetLastError();
}

// levels [lo, hi) of the state (+ optional base / store planes) as a kernel argument
static FlowLevels make_levels(const FlowState& fs, int lo, int hi, const float4* base_f, const float* base_m,
                              float4* out_f, float* out_m, int Hp, int Wp) {
  FlowLevels L{};
  L.mask_replace = fs.mask_replace;
  for (int j = lo; j < hi; ++j) {
    L.f[j - lo] = fs.f[j];
    L.m[j - lo] = fs.m[j];
    L.s[j - lo] = fs.s[j];
    L.hs[j - lo] = Hp / fs.s[j];
    L.ws[j - lo] = Wp / fs.s[j];
    L.inv_s[j - lo] = 1.f / (float)fs.s[j];
  }
  L.base_f = base_f;
  L.base_m = base_m;
  L.out_f = out_f;
  L.out_m = out_m;
  return L;
}

template <typename T>
static void launch_front47_t(int nlev, dim3 g, cudaStream_t st, const uint2* imgs, const uint2* feats,
                             const FlowLevels& L, const BatchTasks& tasks, int Hp, int Wp, int s, void* x) {
  switch (nlev) {
    case 0: VFI_LAUNCH((front47_kernel<T, 0>), g, 128, 0, st, imgs, feats, L, tasks, Hp, Wp, s, (T*)x); break;
    case 1: VFI_LAUNCH((front47_kernel<T, 1>), g, 128, 0, st, imgs, feats, L, tasks, Hp, Wp, s, (T*)x); break;
    case 2: VFI_LAUNCH((front47_kernel<T, 2>), g, 128, 0, st, imgs, feats, L, tasks, Hp, Wp, s, (T*)x); break;
    default: VFI_LAUNCH((front47_kernel<T, 3>), g, 128, 0, st, imgs, feats, L, tasks, Hp, Wp, s, (T*)x); break;
  }
}

template <typename T>
static void launch_front2_t(int nlev, int g, cudaStream_t st, const float4* imgs, const FlowLevels& L,
                            const BatchTasks& tasks, int Hp, int Wp, void* x) {
  switch (nlev) {
    case 1: VFI_LAUNCH((front2_kernel<T, 1>), g, 128, 0, st, imgs, L, tasks, Hp, Wp, (T*)x); break;
    case 2: VFI_LAUNCH((front2_kernel<T, 2>), g, 128, 0, st, imgs, L, tasks, Hp, Wp, (T*)x); break;
    default: VFI_LAUNCH((front2_kernel<T, 3>), g, 128, 0, st, imgs, L, tasks, Hp, Wp, (T*)x); break;
  }
}

template <typename T, int S>
static void launch_front_ts(int nlev, dim3 g, cudaStream_t st, const uint2* imgs, const FlowLevels& L,
                            const BatchTasks& tasks, int Hp, int Wp, int s, void* x) {
  switch (nlev) {
    case 0: VFI_LAUNCH((front_kernel<T, 0, S>), g, 128, 0, st, imgs, L, tasks, Hp, Wp, s, (T*)x); break;
    case 1: VFI_LAUNCH((front_kernel<T, 1, S>), g, 128, 0, st, imgs, L, tasks, Hp, Wp, s, (T*)x); break;
    case 2: VFI_LAUNCH((front_kernel<T, 2, S>), g, 128, 0, st, imgs, L, tasks, Hp, Wp, s, (T*)x); break;
    default: VFI_LAUNCH((front_kernel<T, 3, S>), g, 128, 0, st, imgs, L, tasks, Hp, Wp, s, (T*)x); break;
  }
}

template <typename T>
static void launch_front_t(int nlev, bool shared_taps, dim3 g, cudaStream_t st, const uint2* imgs, const FlowLevels& L,
                           const BatchTasks& tasks, int Hp, int Wp, int s, void* x) {
  if (shared_taps) {
    switch (nlev) {
      case 1: VFI_LAUNCH((front2_kernel<T, 1>), g, 128, 0, st, imgs, L, tasks, Hp, Wp, (T*)x); break;
      case 2: VFI_LAUNCH((front2_kernel<T, 2>), g, 128, 0, st, imgs, L, tasks, Hp, Wp, (T*)x); break;
      default: VFI_LAUNCH((front2_kernel<T, 3>), g, 128, 0, st, imgs, L, tasks, Hp, Wp, (T*)x); break;
    }
  } else if (s == 1) {
    launch_front_ts<T, 1>(nlev, g, st, imgs, L, tasks, Hp, Wp, s, x);  // compile-time scale: 56 instead of 93 registers
  } else {
    launch_front_ts<T, 0>(nlev, g, st, imgs, L, tasks, Hp, Wp, s, x);
  }
}

template <typename T>
static void launch_front417_t(int nlev, dim3 g, cudaStream_t st, const uint2* imgs, const uint4* feats,
                              const FlowLevels& L, const BatchTasks& tasks, int Hp, int Wp, int s, void* x) {
  switch (nlev) {
    case 0: VFI_LAUNCH((front417_kernel<T, 0>), g, 128, 0, st, imgs, feats, L, tasks, Hp, Wp, s, (T*)x); break;
    case 1: VFI_LAUNCH((front417_kernel<T, 1>), g, 128, 0, st, imgs, feats, L, tasks, Hp, Wp, s, (T*)x); break;
    case 2: VFI_LAUNCH((front417_kernel<T, 2>), g, 128, 0, st, imgs, feats, L, tasks, Hp, Wp, s, (T*)x); break;
    default: VFI_LAUNCH((front417_kernel<T, 3>), g, 128, 0, st, imgs, feats, L, tasks, Hp, Wp, s, (T*)x); break;
  }
}

template <typename T>
static void launch_front426_t(int nlev, dim3 g, cudaStream_t st, const uint2* imgs, const uint2* feats,
                              const uint4* prev_feat, int prev_s, const FlowLevels& L, const BatchTasks& tasks, int Hp,
                              int Wp, int s, void* x) {
  switch (nlev) {
    case 0: VFI_LAUNCH((front426_kernel<T, 0>), g, 128, 0, st, imgs, feats, prev_feat, prev_s, L, tasks, Hp, Wp, s, (T*)x); break;
    case 1: VFI_LAUNCH((front426_kernel<T, 1>), g, 128, 0, st, imgs, feats, prev_feat, prev_s, L, tasks, Hp, Wp, s, (T*)x); break;
    case 2: VFI_LAUNCH((front426_kernel<T, 2>), g, 128, 0, st, imgs, feats, prev_feat, prev_s, L, tasks, Hp, Wp, s, (T*)x); break;
    case 3: VFI_LAUNCH((front426_kernel<T, 3>), g, 128, 0, st, imgs, feats, prev_feat, prev_s, L, tasks, Hp, Wp, s, (T*)x); break;
    default: VFI_LAUNCH((front426_kernel<T, 4>), g, 128, 0, st, imgs, feats, prev_feat, prev_s, L, tasks, Hp, Wp, s, (T*)x); break;
  }
}

cudaError_t launch_head0(int op_type, const float4* imgs, const float* w, const float* bias, void* out, int n, int Hp,
                         int Wp, cudaStream_t st) {
  const dim3 g((unsigned)((Wp / 2 + 127) / 128), (unsigned)(Hp / 2), (unsigned)n);
  if (op_type == OP_BF16)
    VFI_LAUNCH((head0_kernel<__nv_bfloat16>), g, 128, 0, st, imgs, w, bias, (__nv_bfloat16*)out, n, Hp, Wp);
  else
    VFI_LAUNCH((head0_kernel<__half>), g, 128, 0, st, imgs, w, bias, (__half*)out, n, Hp, Wp);
  return cudaGetLastError();
}

// block `blk` input: flow = base (if any) + levels [lo, blk); stores the accumulated flow when `store` planes given
cudaError_t launch_encode(const float4* imgs, const float* w0, const float* b0, const float* w1, const float* b1,
                          float* e16, uint2* feats, int n, int Hp, int Wp, cudaStream_t st) {
  const size_t t0 = (size_t)n * (Hp / 2) * (Wp / 2), t1 = (size_t)n * Hp * Wp;
  VFI_LAUNCH((encode_conv_kernel), grid_for(t0, 128), 128, 0, st, imgs, w0, b0, e16, n, Hp, Wp);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  VFI_LAUNCH((encode_deconv_kernel), grid_for(t1, 256), 256, 0, st, e16, w1, b1, feats, n, Hp, Wp);
  return cudaGetLastError();
}

cudaError_t launch_front(int op_type, int arch, const float4* imgs, const uint2* imgs_h, const void* feats, int feat_ch,
                         const void* prev_feat, int prev_s, const FlowState& fs, int blk, int lo, const float4* base_f, const float* base_m, float4* out_f, float* out_m, BatchTasks tasks,
                         int Hp, int Wp, int s, void* x_s2d, cudaStream_t st) {
  const dim3 g((unsigned)((Wp / s + 63) / 64), (unsigned)(Hp / s / 2), (unsigned)tasks.n);  // 64 cells x 2 rows per block
  const FlowLevels L = make_levels(fs, lo, blk, base_f, base_m, out_f, out_m, Hp, Wp);
  const int nlev = (blk == 0) ? 0 : (blk - lo);
  if (blk > 0 && nlev == 0 && base_f == nullptr) return cudaErrorInvalidValue;
  if (nlev > 4 || (arch != 426 && nlev > 3)) return cudaErrorInvalidValue;  // front kernels are built for <= 3 (4.26: 4) levels
  if (arch == 426) {  // 4-channel 16-bit space-to-depth features + the previous block's 8 feature channels
    if (feats == nullptr || (blk > 0 && prev_feat == nullptr)) return cudaErrorInvalidValue;
    if (op_type == OP_BF16)
      launch_front426_t<__nv_bfloat16>(blk == 0 ? 0 : (nlev == 0 ? 1 : nlev), g, st, imgs_h, (const uint2*)feats,
                                       (const uint4*)prev_feat, prev_s, L, tasks, Hp, Wp, s, x_s2d);
    else
      launch_front426_t<__half>(blk == 0 ? 0 : (nlev == 0 ? 1 : nlev), g, st, imgs_h, (const uint2*)feats,
                                (const uint4*)prev_feat, prev_s, L, tasks, Hp, Wp, s, x_s2d);
    return cudaGetLastError();
  }
  if (feats != nullptr && feat_ch == 4) {  // arch 4.7
    if (op_type == OP_BF16)
      launch_front47_t<__nv_bfloat16>(blk == 0 ? 0 : nlev, g, st, imgs_h, (const uint2*)feats, L, tasks, Hp, Wp, s, x_s2d);
    else
      launch_front47_t<__half>(blk == 0 ? 0 : nlev, g, st, imgs_h, (const uint2*)feats, L, tasks, Hp, Wp, s, x_s2d);
    return cudaGetLastError();
  }
  if (feats != nullptr) {  // arch 4.17: 8 feature channels, 16-bit, space-to-depth
    if (op_type == OP_BF16)
      launch_front417_t<__nv_bfloat16>(blk == 0 ? 0 : nlev, g, st, imgs_h, (const uint4*)feats, L, tasks, Hp, Wp, s, x_s2d);
    else
      launch_front417_t<__half>(blk == 0 ? 0 : nlev, g, st, imgs_h, (const uint4*)feats, L, tasks, Hp, Wp, s, x_s2d);
    return cudaGetLastError();
  }
  // scale-2 front without a base plane whose levels are all at scale 4, 8, ...: the level taps are shared per cell
  bool shared_taps = (s == 2 && blk > 0 && base_f == nullptr && nlev >= 1);
  for (int j = 0; j < nlev; ++j) shared_taps = shared_taps && L.s[j] >= 4 && (L.s[j] & (L.s[j] - 1)) == 0;
  const int nl = blk == 0 ? 0 : (nlev == 0 ? 1 : nlev);
  if (op_type == OP_BF16)
    launch_front_t<__nv_bfloat16>(nl, shared_taps, g, st, imgs_h, L, tasks, Hp, Wp, s, x_s2d);
  else
    launch_front_t<__half>(nl, shared_taps, g, st, imgs_h, L, tasks, Hp, Wp, s, x_s2d);
  return cudaGetLastError();
}

cudaError_t launch_materialize(const FlowState& fs, int lo, const float4* base_f, const float* base_m, float4* flow,
                               float* mask, int B, int Hp, int Wp, cudaStream_t st) {
  const size_t total = (size_t)B * Hp * Wp;
  FlowLevels L = make_levels(fs, lo, fs.n, base_f, base_m, nullptr, nullptr, Hp, Wp);
  const int nlev = fs.n - lo;
  switch (nlev) {
    case 1: VFI_LAUNCH((materialize_kernel<1>), grid_for(total, 256), 256, 0, st, L, flow, mask, B, Hp, Wp); break;
    case 2: VFI_LAUNCH((materialize_kernel<2>), grid_for(total, 256), 256, 0, st, L, flow, mask, B, Hp, Wp); break;
    case 3: VFI_LAUNCH((materialize_kernel<3>), grid_for(total, 256), 256, 0, st, L, flow, mask, B, Hp, Wp); break;
    case 4: VFI_LAUNCH((materialize_kernel<4>), grid_for(total, 256), 256, 0, st, L, flow, mask, B, Hp, Wp); break;
    default: VFI_LAUNCH((materialize_kernel<5>), grid_for(total, 256), 256, 0, st, L, flow, mask, B, Hp, Wp); break;
  }
  return cudaGetLastError();
}

cudaError_t launch_final(const float4* imgs, const FlowState& fs, int lo, const float4* base_f, const float* base_m,
                         BatchTasks tasks, int Hp, int Wp, int H, int W, float* out, cudaStream_t st) {
  const FlowLevels L = make_levels(fs, lo, fs.n, base_f, base_m, nullptr, nullptr, Hp, Wp);
  const dim3 g((unsigned)((W + 255) / 256), (unsigned)H, (unsigned)tasks.n);
  switch (fs.n - lo) {
    case 0:  // every level already folded into the dense planes (up-scaled last blocks)
      if (base_f == nullptr) return cudaErrorInvalidValue;
      VFI_LAUNCH((final_kernel<0>), g, 256, 0, st, imgs, L, tasks, Hp, Wp, H, W, out);
      break;
    case 1: VFI_LAUNCH((final_kernel<1>), g, 256, 0, st, imgs, L, tasks, Hp, Wp, H, W, out); break;
    case 2: VFI_LAUNCH((final_kernel<2>), g, 256, 0, st, imgs, L, tasks, Hp, Wp, H, W, out); break;
    case 3: VFI_LAUNCH((final_kernel<3>), g, 256, 0, st, imgs, L, tasks, Hp, Wp, H, W, out); break;
    case 4: VFI_LAUNCH((final_kernel<4>), g, 256, 0, st, imgs, L, tasks, Hp, Wp, H, W, out); break;
    default: VFI_LAUNCH((final_kernel<5>), g, 256, 0, st, imgs, L, tasks, Hp, Wp, H, W, out); break;
  }
  return cudaGetLastError();
}

cudaError_t launch_front_up(int op_type, int arch, const uint2* imgs_h, const void* feats, const void* prev_feat, int prev_s,
                            int prev_k, const float4* F, const float* M, BatchTasks tasks, int Hp, int Wp, int k, void* x_s2d,
                            cudaStream_t st) {
  if ((k != 2 && k != 4) || F == nullptr || M == nullptr || (arch != 46 && arch != 47 && arch != 417 && arch != 426))
    return cudaErrorInvalidValue;
  const dim3 g((unsigned)((Wp * k + 63) / 64), (unsigned)(Hp * k / 2), (unsigned)tasks.n);
  if (arch == 426) {
    if (feats == nullptr || prev_feat == nullptr || prev_s < 1 || prev_k < 1) return cudaErrorInvalidValue;
    if (op_type == OP_BF16)
      VFI_LAUNCH((front_up426_kernel<__nv_bfloat16>), g, 128, 0, st, imgs_h, (const uint2*)feats, (const uint4*)prev_feat, prev_s,
                 prev_k, F, M, tasks, Hp, Wp, k, (__nv_bfloat16*)x_s2d);
    else
      VFI_LAUNCH((front_up426_kernel<__half>), g, 128, 0, st, imgs_h, (const uint2*)feats, (const uint4*)prev_feat, prev_s, prev_k,
                 F, M, tasks, Hp, Wp, k, (__half*)x_s2d);
    return cudaGetLastError();
  }
  if (arch == 417) {
    if (feats == nullptr) return cudaErrorInvalidValue;
    if (op_type == OP_BF16)
      VFI_LAUNCH((front_up417_kernel<__nv_bfloat16>), g, 128, 0, st, imgs_h, (const uint4*)feats, F, M, tasks, Hp, Wp, k,
                 (__nv_bfloat16*)x_s2d);
    else
      VFI_LAUNCH((front_up417_kernel<__half>), g, 128, 0, st, imgs_h, (const uint4*)feats, F, M, tasks, Hp, Wp, k, (__half*)x_s2d);
    return cudaGetLastError();
  }
  if (arch == 47) {
    if (feats == nullptr) return cudaErrorInvalidValue;
    if (op_type == OP_BF16)
      VFI_LAUNCH((front_up47_kernel<__nv_bfloat16>), g, 128, 0, st, imgs_h, (const uint2*)feats, F, M, tasks, Hp, Wp, k,
                 (__nv_bfloat16*)x_s2d);
    else
      VFI_LAUNCH((front_up47_kernel<__half>), g, 128, 0, st, imgs_h, (const uint2*)feats, F, M, tasks, Hp, Wp, k, (__half*)x_s2d);
    return cudaGetLastError();
  }
  if (op_type == OP_BF16)
    VFI_LAUNCH((front_up_kernel<__nv_bfloat16>), g, 128, 0, st, imgs_h, F, M, tasks, Hp, Wp, k, (__nv_bfloat16*)x_s2d);
  else
    VFI_LAUNCH((front_up_kernel<__half>), g, 128, 0, st, imgs_h, F, M, tasks, Hp, Wp, k, (__half*)x_s2d);
  return cudaGetLastError();
}

cudaError_t launch_fold_down(const float4* tf, const float* tm, int k, float4* F, float* M, int B, int Hp, int Wp,
                             int mask_replace, cudaStream_t st) {
  if (k != 2 && k != 4) return cudaErrorInvalidValue;
  VFI_LAUNCH((fold_down_kernel), grid_for((size_t)B * Hp * Wp, 256), 256, 0, st, tf, tm, k, F, M, B, Hp, Wp, mask_replace);
  return cudaGetLastError();
}

cudaError_t launch_warp(const float* img, const float* flow, float* out, int B, int H, int W, int C, cudaStream_t st) {
  if (C % 4 == 0) {
    const size_t total = (size_t)B * H * W * (C / 4);
    VFI_LAUNCH((warp_kernel<4>), grid_for(total, 256), 256, 0, st, img, flow, out, B, H, W, C);
  } else {
    const size_t total = (size_t)B * H * W * C;
    VFI_LAUNCH((warp_kernel<1>), grid_for(total, 256), 256, 0, st, img, flow, out, B, H, W, C);
  }
  return cudaGetLastError();
}

}  // namespace vfi
