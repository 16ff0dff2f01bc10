// IFRNet-S / IFRNet-L on H100: weight repacking, channel layout, workspace, the forward schedule and its C ABI
// (include/vfi_b200.h).  Reference: vfi_models/ifrnet/IFRNet_{S,L}_arch.py, ifrnet/__init__.py.
//
// Every convolution but the 3-channel first one is a streamconv layer with the IFRNet epilogue (ext 2): + bias
// (+ residual) -> PReLU with one slope per channel (slope 1 = none) -> 16-bit, the first n_f32 columns to an fp32 tensor.
//   prep, first_conv (CUDA cores)   mean_, resize by t, pyramid1.0 (3x3 / 7x7, stride 2) + PReLU
//   pyramid1.1 .. pyramid4.1        3x3 convs; pyramidN.0 (stride 2) as a 2x2 conv over the space-to-depth copy
//   decoder d (4, 3, 2, 1)          input (dec4_in / dec_in: warps at the feature's own size), convrelu, ResBlock,
//                                   ConvTranspose2d(4, 2, 1) as four 2x2 phase convs: flow (mask, res) columns fp32
//   final (CUDA cores)              resize by 1/t, image warps, merge, clamp, crop
//
// Channel layout.  streamconv reads 64-channel k-blocks from at most two sources, so each group a conv reads or writes
// on its own starts on a 64-channel boundary; padding channels hold zeros and meet zero weights:
//   encoder level l           [C_l, pad to 64]                     (the space-to-depth copy: phase q at q * up8(C))
//   ResBlock tensors (C, s)   [C - s main, pad to 64 | s side, pad to 64]: conv2 / conv4 read the side slice and write
//                             a separate tensor (neighbouring tiles still read its halo); conv3 / conv5 read
//                             cat(main slice, that tensor) as their two sources
//   decoder 4 input           [f0_4 | f1_4 | embt]                 each group padded to 64
//   decoder 3..1 input        [ft_ | warp(f0) | warp(f1) | flow0, flow1]
//   ConvT phase columns       [flow0, flow1 (fp32) | 4 zero | ft_ ...]; decoder 1: [flow0, flow1, mask, res] all fp32
// The packer maps each physical channel to its logical one (-1: padding).
#include <cuda_fp16.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <functional>
#include <string>

#include "../../include/vfi_b200.h"
#include "vfi_internal.h"

namespace vfi {

namespace {

constexpr int kDecBase = 10;   // layer id of decoder k (0 = decoder4 .. 3 = decoder1): 10 + 10 k + {0 conv0, 1..5
constexpr int kNumLayers = 50; // ResBlock conv1..conv5, 6..9 ConvT phase py * 2 + px}; encoder 0 .. 6

struct Arch {
  int enc[4];   // pyramid channels
  int side;     // ResBlock side channels
  int k0;       // first conv kernel (stride 2, padding k0 / 2)
  int dc[4];    // decoder4..1 convblock channels
  int dout[4];  // decoder4..1 ConvT outputs
};
const Arch kArchS = {{24, 36, 54, 72}, 24, 3, {144, 162, 108, 72}, {58, 40, 28, 8}};
const Arch kArchL = {{64, 96, 144, 192}, 64, 7, {384, 432, 288, 192}, {148, 100, 68, 8}};

int up64(int v) { return (v + 63) / 64 * 64; }
int up16(int v) { return (v + 15) / 16 * 16; }
int up8(int v) { return (v + 7) / 8 * 8; }

using Map = std::vector<int>;  // physical channel -> logical channel (-1: padding)
Map map_plain(int C) {
  Map m(up64(C));
  for (int j = 0; j < (int)m.size(); ++j) m[j] = j < C ? j : -1;
  return m;
}
// ResBlock layout: main channels [0, C - s) at 0, side channels at up64(C - s)
Map map_split(int C, int s) {
  const int M = up64(C - s);
  Map m(M + up64(s), -1);
  for (int j = 0; j < C - s; ++j) m[j] = j;
  for (int i = 0; i < s; ++i) m[M + i] = C - s + i;
  return m;
}
// groups of the given sizes at 64-aligned offsets, logical channels in order
Map map_groups(std::initializer_list<int> sizes) {
  Map m;
  int lo = 0;
  for (int n : sizes) {
    const size_t at = m.size();
    m.resize(at + up64(n), -1);
    for (int i = 0; i < n; ++i) m[at + i] = lo + i;
    lo += n;
  }
  return m;
}
// the space-to-depth copy of a C-channel tensor: phase q at q * up8(C); logical index q * C + c
Map map_s2d(int C) {
  const int cq = up8(C);
  Map m(up64(4 * cq), -1);
  for (int q = 0; q < 4; ++q)
    for (int c = 0; c < C; ++c) m[q * cq + c] = q * C + c;
  return m;
}

struct IBuf {
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t ensure(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e == cudaSuccess) cap = bytes;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};

}  // namespace

struct IfrnetState : ModelState {
  int op_type = OP_F16;
  bool loaded = false;
  bool use_ref = false;  // debug: every conv through the CUDA-core checker
  int variant = 0;       // 0: IFRNet-S, 1: IFRNet-L
  Arch a{};
  std::vector<void*> allocs;
  float* w0 = nullptr;  // pyramid1.0: [C][3][k][k], bias, slopes
  float* b0 = nullptr;
  float* s0 = nullptr;
  StreamConvLayer conv[kNumLayers];
  // workspace
  IBuf partial, mean, xin, t1, enc[4], s2d, fin, x, ra, rb, sd, ph16, ph32, accA, accB;
  ~IfrnetState() override {
    for (void* p : allocs) cudaFree(p);
    for (IBuf* b : {&partial, &mean, &xin, &t1, &enc[0], &enc[1], &enc[2], &enc[3], &s2d, &fin, &x, &ra, &rb, &sd, &ph16,
                    &ph32, &accA, &accB})
      b->release();
  }
};

namespace {

IfrnetState* state(vfi_ctx* c) { return c ? static_cast<IfrnetState*>(ctx_ifrnet(c)) : nullptr; }

#define ICK(call)                                                            \
  do {                                                                       \
    cudaError_t _e = (call);                                                 \
    if (_e != cudaSuccess) {                                                 \
      set_error(std::string(#call) + ": " + cudaGetErrorString(_e));         \
      return VFI_E_CUDA;                                                     \
    }                                                                        \
  } while (0)

#define IRUN(expr)           \
  do {                       \
    const int _rc = (expr);  \
    if (_rc) return _rc;     \
  } while (0)

int ifail(int code, const std::string& msg) {
  set_error(msg);
  return code;
}

template <class T>
int iupload(IfrnetState* f, const T* h, size_t n, void** dptr) {
  void* d = nullptr;
  ICK(cudaMalloc(&d, n * sizeof(T)));
  f->allocs.push_back(d);
  ICK(cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice));
  *dptr = d;
  return VFI_OK;
}

// Packs one layer: input channels in_map (c0 from source 0, the rest from source 1), output columns out_map;
// wfun(logical output, tap, logical input), bias and PReLU slopes by logical output (slopes nullptr: identity)
int build_layer(IfrnetState* f, StreamConvLayer& L, int ksize, const Map& in_map, int c0, const Map& out_map,
                const std::function<float(int, int, int)>& wfun, const float* bias, const float* slopes, int n_f32) {
  L = StreamConvLayer{};
  L.ksize = ksize;
  L.c0 = c0;
  L.c1 = (int)in_map.size() - c0;
  L.n_total = (int)out_map.size();
  L.act = 0;
  L.ext = 2;
  L.n_f32 = n_f32;
  std::vector<uint16_t> pk;
  StreamConvParams p{};
  if (!pack_streamconv(L, f->op_type, [&](int n, int tap, int j) -> float {
        const int lo = out_map[n], li = in_map[j];
        return (lo < 0 || li < 0) ? 0.f : wfun(lo, tap, li);
      }, &pk, &p))
    return ifail(VFI_E_INVALID, "ifrnet: layer shape not supported by streamconv");
  std::vector<float> sh(L.n_total, 0.f), sl(L.n_total, 1.f);
  for (int n = 0; n < L.n_total; ++n) {
    const int lo = out_map[n];
    if (lo < 0) continue;
    sh[n] = bias[lo];
    if (slopes) sl[n] = slopes[lo];
  }
  void* d = nullptr;
  IRUN(iupload(f, pk.data(), pk.size(), &d));
  L.w = d;
  IRUN(iupload(f, sh.data(), sh.size(), &d));
  L.shift = static_cast<float*>(d);
  IRUN(iupload(f, sl.data(), sl.size(), &d));
  L.slopes = static_cast<float*>(d);
  return VFI_OK;
}

// Conv2d(cin, cout, 3, 1, 1) weight [cout][cin][3][3]
int build_conv3(IfrnetState* f, StreamConvLayer& L, const Map& in_map, int c0, const Map& out_map, int cin, const float* w,
                const float* b, const float* slopes) {
  return build_layer(f, L, 3, in_map, c0, out_map, [&](int lo, int tap, int li) { return w[((size_t)lo * cin + li) * 9 + tap]; },
                     b, slopes, 0);
}

// Conv2d(cin, cout, 3, stride 2, padding 1) as a 2x2 conv over the space-to-depth copy (logical input q * cin + c):
// tap d (0 / 1) of an axis reads offset d - 1, i.e. kernel index 0 (d = 0, phase 1), 1 (d = 1, phase 0), 2 (d = 1, phase 1)
int build_conv_s2(IfrnetState* f, StreamConvLayer& L, int cin, int cout, const float* w, const float* b, const float* slopes) {
  const int r = build_layer(f, L, 2, map_s2d(cin), (int)map_s2d(cin).size(), map_plain(cout), [&](int lo, int tap, int li) -> float {
    const int q = li / cin, c = li - q * cin, py = q >> 1, px = q & 1, dy = tap >> 1, dx = tap & 1;
    const int ky = dy == 0 ? (py ? 0 : -1) : 1 + py, kx = dx == 0 ? (px ? 0 : -1) : 1 + px;
    if (ky < 0 || kx < 0) return 0.f;
    return w[((size_t)lo * cin + c) * 9 + ky * 3 + kx];
  }, b, slopes, 0);
  L.pad_before = 1;
  return r;
}

// the ConvT's output columns: [flow0, flow1 | 4 zero | ft_] (fp32 columns 0..3), decoder 1: [8 outputs] all fp32
Map map_convt_out(int cout, bool last) {
  Map m(last ? 16 : up16(8 + cout - 4), -1);
  if (last) {
    for (int i = 0; i < 8; ++i) m[i] = i;
  } else {
    for (int i = 0; i < 4; ++i) m[i] = i;
    for (int i = 4; i < cout; ++i) m[4 + i] = i;
  }
  return m;
}

// ConvTranspose2d(cin, cout, 4, 2, 1) weight [cin][cout][4][4]: output row 2 i + py sums input rows i + d - (1 - py),
// d = 0, 1, with kernel row 3 - py - 2 d.  Phase (py, px) = a 2x2 conv with (1 - py, 1 - px) padding rows / columns before.
int build_convT_phase(IfrnetState* f, StreamConvLayer& L, const Map& in_map, int cout, bool last, int py, int px,
                      const float* w, const float* b) {
  const int r = build_layer(f, L, 2, in_map, (int)in_map.size(), map_convt_out(cout, last), [&](int lo, int tap, int li) {
    const int ky = 3 - py - 2 * (tap >> 1), kx = 3 - px - 2 * (tap & 1);
    return w[(((size_t)li * cout + lo) * 4 + ky) * 4 + kx];
  }, b, nullptr, last ? 8 : 4);
  L.pad_before = 1 - py;
  L.pad_before_x = 1 - px;
  return r;
}

// the decoder inputs' layouts (decoder k = 0 is decoder 4)
Map dec_in_map(const Arch& a, int k) {
  if (k == 0) return map_groups({a.enc[3], a.enc[3], 1});
  const int ft = a.dout[k - 1] - 4, cf = a.enc[3 - k];
  return map_groups({ft, cf, cf, 4});
}

// ---------------------------------------------------------------- geometry
struct Geo {
  int H, W, Hp, Wp;
  int h[5], w[5];  // h[0]: the resized input; h[1..4]: pyramid levels (ceil halving)
  int gh[4], gw[4];  // decoder k runs on gh[k] x gw[k] (k = 0: decoder 4 on level 4; then doubling)
  int hq, wq;      // decoder 1's output grid
  int hF, wF;      // the final resize's size (cropped to H x W)
  float s_in, s_out, fmul;  // resize scales passed to the kernels (1 / scale_factor) and the flow multiplier 1 / t
};

// sizes with the reference's own arithmetic: F.interpolate(scale_factor=s) gives floor(n * s) (double), a stride-2
// conv ceil(n / 2), a ConvT 2 n
int geometry(int H, int W, double t, Geo* g) {
  if (!(t > 0.0) || !std::isfinite(t)) return ifail(VFI_E_INVALID, "ifrnet: the resize factor must be a positive number");
  g->H = H;
  g->W = W;
  g->Hp = ((H - 1) / 64 + 1) * 64;
  g->Wp = ((W - 1) / 64 + 1) * 64;
  const double h0 = std::floor((double)g->Hp * t), w0 = std::floor((double)g->Wp * t);
  if (h0 < 1.0 || w0 < 1.0)
    return ifail(VFI_E_INVALID, "ifrnet: the resize factor " + std::to_string(t) + " gives an empty encoder input");
  if (h0 > 65536.0 || w0 > 65536.0) return ifail(VFI_E_INVALID, "ifrnet: the resize factor gives a too large encoder input");
  g->h[0] = (int)h0;
  g->w[0] = (int)w0;
  for (int l = 1; l <= 4; ++l) {
    g->h[l] = (g->h[l - 1] + 1) / 2;
    g->w[l] = (g->w[l - 1] + 1) / 2;
  }
  g->gh[0] = g->h[4];
  g->gw[0] = g->w[4];
  for (int k = 1; k < 4; ++k) {
    g->gh[k] = 2 * g->gh[k - 1];
    g->gw[k] = 2 * g->gw[k - 1];
  }
  g->hq = 2 * g->gh[3];
  g->wq = 2 * g->gw[3];
  const double inv = 1.0 / t;
  const double hF = std::floor((double)g->hq * inv), wF = std::floor((double)g->wq * inv);
  if (hF < (double)H || wF < (double)W)
    return ifail(VFI_E_INVALID, "ifrnet: the resize factor " + std::to_string(t) + " gives a " + std::to_string((long long)hF) +
                                    " x " + std::to_string((long long)wF) + " output, smaller than the frame");
  g->hF = (int)hF;
  g->wF = (int)wF;
  g->s_in = (float)(1.0 / t);
  g->s_out = (float)(1.0 / inv);
  g->fmul = (float)inv;
  return VFI_OK;
}

uint8_t* bp(const IBuf& b) { return static_cast<uint8_t*>(b.p); }

int ensure_workspace(IfrnetState* f, const Geo& g) {
  const Arch& a = f->a;
  const size_t e = 2;
  ICK(f->partial.ensure(sizeof(double) * ifrnet_sum_blocks()));
  ICK(f->mean.ensure(sizeof(float)));
  ICK(f->xin.ensure((size_t)2 * g.h[0] * g.w[0] * 16));
  size_t s2d = 0, t1 = (size_t)2 * g.h[1] * g.w[1] * 64 * e;  // t1: the first conv's output, then each stride-2 conv's
  for (int l = 0; l < 4; ++l) {
    const size_t px = (size_t)2 * g.h[l + 1] * g.w[l + 1];
    ICK(f->enc[l].ensure(px * up64(a.enc[l]) * e));
    if (l > 0) {
      s2d = std::max(s2d, px * map_s2d(a.enc[l - 1]).size() * e);
      t1 = std::max(t1, px * up64(a.enc[l]) * e);
    }
  }
  ICK(f->t1.ensure(t1));
  ICK(f->s2d.ensure(s2d));
  size_t fin = 0, res = 0, sd = 0, p16 = 0, p32 = 0, acc = 0;
  for (int k = 0; k < 4; ++k) {
    const size_t px = (size_t)g.gh[k] * g.gw[k];
    fin = std::max(fin, px * dec_in_map(a, k).size() * e);
    res = std::max(res, px * map_split(a.dc[k], a.side).size() * e);
    sd = std::max(sd, px * 64 * e);
    p16 = std::max(p16, px * 4 * map_convt_out(a.dout[k], k == 3).size() * e);
    p32 = std::max(p32, px * 4 * (k == 3 ? 8 : 4) * 4);
    acc = std::max(acc, 4 * px * (k == 3 ? 8 : 4) * 4);
  }
  ICK(f->fin.ensure(fin));
  for (IBuf* b : {&f->x, &f->ra, &f->rb}) ICK(b->ensure(res));
  ICK(f->sd.ensure(sd));
  ICK(f->ph16.ensure(p16));
  ICK(f->ph32.ensure(p32));
  ICK(f->accA.ensure(acc));
  ICK(f->accB.ensure(acc));
  return VFI_OK;
}

struct Runner {
  IfrnetState* f;
  CtxInfo ci;
  cudaStream_t st;
  int launches = 0;
  int ck(cudaError_t e, const char* what) {
    ++launches;
    if (e != cudaSuccess) {
      set_error(std::string("ifrnet: ") + what + ": " + cudaGetErrorString(e) + " / " + vfi_last_error());
      return VFI_E_CUDA;
    }
    return VFI_OK;
  }
  int conv(int id, const void* s0, int p0, const void* s1, int p1, void* out, int op, int B, int H, int W,
           const void* res = nullptr, float* o32 = nullptr, int p32 = 0) {
    return ck(launch_streamconv(f->conv[id], f->op_type, s0, p0, s1, p1, out, op, B, H, W, ci.num_sms, f->use_ref, st, res,
                                o32, p32),
              "streamconv");
  }
};

int forward(vfi_ctx* c, IfrnetState* f, const float* img0, const float* img1, const Geo& g, float embt, float* out,
            cudaStream_t st) {
  IRUN(ensure_workspace(f, g));
  const Arch& a = f->a;
  const int op = f->op_type;
  Runner r{f, ctx_info(c), st};
  // ---- mean_, resize, encoder (IRFNet.forward, Encoder.forward; both frames as one batch of two)
  IRUN(r.ck(launch_ifrnet_mean(img0, img1, g.H, g.W, g.Hp, g.Wp, (double*)f->partial.p, (float*)f->mean.p, st), "mean"));
  IRUN(r.ck(launch_ifrnet_prep(img0, img1, g.H, g.W, g.Hp, g.Wp, g.h[0], g.w[0], g.s_in, (const float*)f->mean.p,
                               (float4*)f->xin.p, st),
            "prep"));
  IRUN(r.ck(launch_ifrnet_first_conv(op, (const float4*)f->xin.p, g.h[0], g.w[0], g.h[1], g.w[1], a.k0, f->w0, f->b0, f->s0,
                                     a.enc[0], 64, f->t1.p, st),
            "first_conv"));
  IRUN(r.conv(0, f->t1.p, 64, nullptr, 0, f->enc[0].p, up64(a.enc[0]), 2, g.h[1], g.w[1]));
  for (int l = 1; l < 4; ++l) {
    const int Pi = up64(a.enc[l - 1]), Ps = (int)map_s2d(a.enc[l - 1]).size(), Po = up64(a.enc[l]);
    IRUN(r.ck(launch_ifrnet_s2d(op, f->enc[l - 1].p, Pi, up8(a.enc[l - 1]), 2, g.h[l], g.w[l], f->s2d.p, Ps, st), "s2d"));
    IRUN(r.conv(2 * l - 1, f->s2d.p, Ps, nullptr, 0, f->t1.p, Po, 2, g.h[l + 1], g.w[l + 1]));
    IRUN(r.conv(2 * l, f->t1.p, Po, nullptr, 0, f->enc[l].p, Po, 2, g.h[l + 1], g.w[l + 1]));
  }
  // ---- decoders 4 .. 1
  for (int k = 0; k < 4; ++k) {
    const int gh = g.gh[k], gw = g.gw[k], id = kDecBase + 10 * k;
    const int PI = (int)dec_in_map(a, k).size(), C = a.dc[k], M = up64(C - a.side), PR = M + up64(a.side);
    if (k == 0) {
      IRUN(r.ck(launch_ifrnet_dec4_in(op, f->enc[3].p, up64(a.enc[3]), up64(a.enc[3]), gh, gw, embt, f->fin.p, st), "dec4_in"));
    } else {
      const int ft = a.dout[k - 1] - 4, cf = a.enc[3 - k], lv = 4 - k;  // features of pyramid level 4 - k
      const int g1 = up64(ft), g2 = g1 + up64(cf), g3 = g2 + up64(cf);
      const int pp = (int)map_convt_out(a.dout[k - 1], false).size();
      const float* acc = (const float*)(k % 2 ? f->accA.p : f->accB.p);
      IRUN(r.ck(launch_ifrnet_dec_in(op, f->ph16.p, pp, f->enc[lv - 1].p, up64(cf), g.h[lv], g.w[lv], acc, gh, gw, g1, g2, g3,
                                     f->fin.p, st),
                "dec_in"));
    }
    // convrelu, ResBlock (conv2 / conv4 write the side tensor sd), ConvT phases
    IRUN(r.conv(id, f->fin.p, PI, nullptr, 0, f->x.p, PR, 1, gh, gw));
    IRUN(r.conv(id + 1, f->x.p, PR, nullptr, 0, f->ra.p, PR, 1, gh, gw));
    IRUN(r.conv(id + 2, bp(f->ra) + (size_t)M * 2, PR, nullptr, 0, f->sd.p, 64, 1, gh, gw));
    IRUN(r.conv(id + 3, f->ra.p, PR, f->sd.p, 64, f->rb.p, PR, 1, gh, gw));
    IRUN(r.conv(id + 4, bp(f->rb) + (size_t)M * 2, PR, nullptr, 0, f->sd.p, 64, 1, gh, gw));
    IRUN(r.conv(id + 5, f->rb.p, PR, f->sd.p, 64, f->ra.p, PR, 1, gh, gw, f->x.p));
    const bool last = k == 3;
    const int NT = (int)map_convt_out(a.dout[k], last).size(), nf = last ? 8 : 4;
    for (int q = 0; q < 4; ++q)
      IRUN(r.conv(id + 6 + q, f->ra.p, PR, nullptr, 0, bp(f->ph16) + (size_t)q * NT * 2, 4 * NT, 1, gh, gw, nullptr,
                  (float*)f->ph32.p + (size_t)q * nf, 4 * nf));
    // flows on the doubled grid: decoder 4 writes accA, then B, A, B
    float* acc_out = (float*)(k % 2 ? f->accB.p : f->accA.p);
    const float* acc_prev = k == 0 ? nullptr : (const float*)(k % 2 ? f->accA.p : f->accB.p);
    IRUN(r.ck(launch_ifrnet_dec_flow((const float*)f->ph32.p, nf, acc_prev, gh, gw, acc_out, st), "dec_flow"));
  }
  IRUN(r.ck(launch_ifrnet_final(img0, img1, g.H, g.W, g.Hp, g.Wp, (const float*)f->accB.p, g.hq, g.wq, g.hF, g.wF, g.s_out,
                                g.fmul, (const float*)f->mean.p, out, st),
            "final"));
  ctx_add_launches(c, r.launches);
  return VFI_OK;
}

}  // namespace
}  // namespace vfi

using namespace vfi;

extern "C" {

/* tensor order: IRFNet_S / IRFNet_L .state_dict() (engine.py ifrnet_state_dict_spec) */
int vfi_ifrnet_load(vfi_ctx* c, const float* const* T, const int64_t* numel, int n_tensors, int operand_type) {
  if (!c || !T || !numel) return ifail(VFI_E_INVALID, "null argument");
  if (n_tensors != VFI_IFRNET_NUM_TENSORS) return ifail(VFI_E_INVALID, "ifrnet: expected 104 tensors");
  if (operand_type != VFI_OPERAND_F16 && operand_type != VFI_OPERAND_BF16) return ifail(VFI_E_INVALID, "operand type");
  const bool large = numel[0] == 64LL * 3 * 49;
  if (!large && numel[0] != 24LL * 3 * 9)
    return ifail(VFI_E_INVALID, "ifrnet: encoder.pyramid1.0.0.weight is neither IFRNet-S's nor IFRNet-L's");
  const CtxInfo ci = ctx_info(c);
  ICK(cudaSetDevice(ci.device));
  delete ctx_ifrnet(c);
  IfrnetState* f = new IfrnetState();
  ctx_ifrnet(c) = f;
  f->op_type = operand_type;
  f->variant = large ? 1 : 0;
  f->a = large ? kArchL : kArchS;
  const Arch& a = f->a;
  int t = 0;
  bool sizes_ok = true;
  auto take = [&](int64_t n) -> const float* {
    if (t >= n_tensors || numel[t] != n) sizes_ok = false;
    return sizes_ok ? T[t++] : nullptr;
  };
  auto bad = [&](const std::string& what) {
    return ifail(VFI_E_INVALID, "ifrnet: tensor " + std::to_string(t) + " (" + what + ") has " +
                                    std::to_string((long long)(t < n_tensors ? numel[t] : -1)) +
                                    " elements, not what IFRNet-" + (large ? "L" : "S") + " has");
  };
  void* d = nullptr;
  // ---- encoder.pyramid{1..4}.{0,1}: .0.weight, .0.bias, .1.weight (PReLU)
  int cin = 3;
  for (int l = 0; l < 4; ++l) {
    const int Co = a.enc[l];
    for (int j = 0; j < 2; ++j) {
      const int ks = (l == 0 && j == 0) ? a.k0 : 3, ci_ = j == 0 ? cin : Co;
      const float* w = take((int64_t)Co * ci_ * ks * ks);
      const float* b = take(Co);
      const float* s = take(Co);
      if (!sizes_ok) return bad("encoder.pyramid" + std::to_string(l + 1) + "." + std::to_string(j));
      if (l == 0 && j == 0) {
        IRUN(iupload(f, w, (size_t)Co * 3 * ks * ks, &d));
        f->w0 = (float*)d;
        IRUN(iupload(f, b, Co, &d));
        f->b0 = (float*)d;
        IRUN(iupload(f, s, Co, &d));
        f->s0 = (float*)d;
      } else if (j == 0) {
        IRUN(build_conv_s2(f, f->conv[2 * l - 1], ci_, Co, w, b, s));
      } else {
        IRUN(build_conv3(f, f->conv[l == 0 ? 0 : 2 * l], map_plain(Co), up64(Co), map_plain(Co), Co, w, b, s));
      }
    }
    cin = Co;
  }
  // ---- decoder4 .. decoder1: convblock.0 (convrelu), convblock.1 (ResBlock), convblock.2 (ConvTranspose2d)
  for (int k = 0; k < 4; ++k) {
    const int id = kDecBase + 10 * k, C = a.dc[k], s = a.side, M = up64(C - s);
    const Map in = dec_in_map(a, k), sp = map_split(C, s), side = map_plain(s);
    int cin0 = 0;
    for (int v : in) cin0 = std::max(cin0, v + 1);
    const std::string name = "decoder" + std::to_string(4 - k);
    const float* w = take((int64_t)C * cin0 * 9);
    const float* b = take(C);
    const float* sl = take(C);
    if (!sizes_ok) return bad(name + ".convblock.0");
    IRUN(build_conv3(f, f->conv[id], in, (int)in.size(), sp, cin0, w, b, sl));
    // ResBlock: conv1 .. conv4 (conv + PReLU), conv5, prelu
    const float* rw[5];
    const float* rbias[5];
    const float* rsl[5];
    for (int j = 0; j < 5; ++j) {  // conv1 .. conv4: .0.weight, .0.bias, .1.weight; conv5: weight, bias; then prelu
      const int n = (j == 1 || j == 3) ? s : C;
      rw[j] = take((int64_t)n * n * 9);
      rbias[j] = take(n);
      rsl[j] = take(n);
      if (!sizes_ok) return bad(name + ".convblock.1." + (j == 4 ? std::string("prelu") : "conv" + std::to_string(j + 1)));
    }
    IRUN(build_conv3(f, f->conv[id + 1], sp, (int)sp.size(), sp, C, rw[0], rbias[0], rsl[0]));
    IRUN(build_conv3(f, f->conv[id + 2], side, 64, side, s, rw[1], rbias[1], rsl[1]));
    IRUN(build_conv3(f, f->conv[id + 3], sp, M, sp, C, rw[2], rbias[2], rsl[2]));
    IRUN(build_conv3(f, f->conv[id + 4], side, 64, side, s, rw[3], rbias[3], rsl[3]));
    IRUN(build_conv3(f, f->conv[id + 5], sp, M, sp, C, rw[4], rbias[4], rsl[4]));
    const float* tw = take((int64_t)C * a.dout[k] * 16);
    const float* tb = take(a.dout[k]);
    if (!sizes_ok) return bad(name + ".convblock.2");
    for (int q = 0; q < 4; ++q)
      IRUN(build_convT_phase(f, f->conv[id + 6 + q], sp, a.dout[k], k == 3, q >> 1, q & 1, tw, tb));
  }
  if (t != n_tensors) return ifail(VFI_E_INVALID, "ifrnet: unused tensors");
  f->loaded = true;
  return VFI_OK;
}

int vfi_ifrnet_forward(vfi_ctx* c, const float* img0, const float* img1, int H, int W, double t, double embt, float* out,
                       void* stream) {
  if (!c || !img0 || !img1 || !out) return ifail(VFI_E_INVALID, "null argument");
  IfrnetState* f = state(c);
  if (!f || !f->loaded) return ifail(VFI_E_STATE, "vfi_ifrnet_load has not been called");
  if (H < 1 || W < 1) return ifail(VFI_E_INVALID, "ifrnet: empty frames");
  if (!std::isfinite(embt)) return ifail(VFI_E_INVALID, "ifrnet: embt must be finite");
  Geo g{};
  IRUN(geometry(H, W, t, &g));
  ICK(cudaSetDevice(ctx_info(c).device));
  return forward(c, f, img0, img1, g, (float)embt, out, static_cast<cudaStream_t>(stream));
}

int vfi_ifrnet_geometry(int H, int W, double t, int32_t* info, int cap) {
  if (!info || H < 1 || W < 1) return ifail(VFI_E_INVALID, "ifrnet: bad geometry arguments");
  Geo g{};
  IRUN(geometry(H, W, t, &g));
  const int32_t v[22] = {g.Hp, g.Wp, g.h[0], g.w[0], g.h[1], g.w[1], g.h[2], g.w[2], g.h[3], g.w[3], g.h[4], g.w[4],
                         g.gh[1], g.gw[1], g.gh[2], g.gw[2], g.gh[3], g.gw[3], g.hq, g.wq, g.hF, g.wF};
  for (int i = 0; i < cap && i < 22; ++i) info[i] = v[i];
  return VFI_OK;
}

int vfi_ifrnet_debug_set_ref(vfi_ctx* c, int use_ref) {
  IfrnetState* f = state(c);
  if (!f) return ifail(VFI_E_STATE, "vfi_ifrnet_load has not been called");
  f->use_ref = use_ref != 0;
  return VFI_OK;
}

static const StreamConvLayer* ifrnet_layer(vfi_ctx* c, int layer) {
  IfrnetState* f = state(c);
  if (!f || !f->loaded || layer < 0 || layer >= kNumLayers || !f->conv[layer].w) return nullptr;
  return &f->conv[layer];
}

int vfi_ifrnet_debug_conv(vfi_ctx* c, int layer, const void* src0, int pitch0, const void* src1, int pitch1, void* out,
                          int out_pitch, const void* res, float* out_f32, int f32_pitch, int B, int H, int W, int impl,
                          void* stream) {
  const StreamConvLayer* L = ifrnet_layer(c, layer);
  if (!L) return ifail(VFI_E_INVALID, "ifrnet: no such conv layer (or weights not loaded)");
  ICK(cudaSetDevice(ctx_info(c).device));
  const cudaError_t e = launch_streamconv(*L, state(c)->op_type, src0, pitch0, src1, pitch1, out, out_pitch, B, H, W,
                                          ctx_info(c).num_sms, impl != 0, static_cast<cudaStream_t>(stream), res, out_f32,
                                          f32_pitch);
  ctx_add_launches(c, 1);
  if (e != cudaSuccess) return ifail(VFI_E_CUDA, std::string("streamconv: ") + cudaGetErrorString(e) + " / " + vfi_last_error());
  return VFI_OK;
}

int vfi_ifrnet_layer_plan(vfi_ctx* c, int layer, int32_t* info, int cap) {
  const StreamConvLayer* L = ifrnet_layer(c, layer);
  if (!L || !info) return ifail(VFI_E_INVALID, "ifrnet: no such conv layer (or weights not loaded)");
  StreamConvParams p{};
  if (!streamconv_plan(*L, &p)) return ifail(VFI_E_INVALID, "ifrnet: plan failed");
  const int32_t v[12] = {L->c0, L->c1, L->n_total, L->ksize, -p.halo_y0, -p.halo_x0, p.n_cta, p.nsplit, p.a_slots,
                         p.b_slots, (int32_t)p.smem_bytes, L->n_f32};
  for (int i = 0; i < cap && i < 12; ++i) info[i] = v[i];
  return VFI_OK;
}

int vfi_ifrnet_info(vfi_ctx* c, int* variant) {
  IfrnetState* f = state(c);
  if (!f || !f->loaded) return ifail(VFI_E_STATE, "vfi_ifrnet_load has not been called");
  if (variant) *variant = f->variant;
  return VFI_OK;
}

}  // extern "C"
