// FLAVR (UNet_3D_3D "unet_18", n_inputs 4) on H100: weight repacking, workspace, the forward schedule and its C ABI
// (include/vfi_b200.h).  Reference: vfi_models/flavr/flavr_arch.py, resnet_3D.py, flavr/__init__.py.
//
// Activations are 16-bit [image][h][w][C] tensors with image = window * 4 + plane; a 3x3x3 conv is a streamconv layer
// with three temporal taps over the four planes of its window (zero planes outside).  H2 = Hp / 2 etc.
//   frame_sums, prep, stem              replicate pad, mean subtraction, Conv3d(3,64,(3,7,7),s(1,2,2)) + ReLU  (CUDA cores)
//   layer1..4, two BasicBlocks each     conv1 (+ ReLU in the epilogue), conv2, gate, x * g + residual -> ReLU
//                                       layer2 / layer3 block 0: stride (1,2,2) as a 2x2(x3) conv over the space-to-depth
//                                       copy of the previous output; the 1x1x1 downsample reads its phase-(0,0) slice
//   decoder 0, 3                        3x3x3 conv on cat(previous, skip) (two sources), gate, LeakyReLU(0.2)
//   decoder 1, 2, 4                     ConvTranspose3d((3,4,4), s(1,2,2), p1) as four 2x2(x3) phase convs, gate, and the
//                                       depth-to-space interleave of the phases, LeakyReLU(0.2)
//   feature_fuse                        cat(unbind(T)) + 1x1 conv = a streamconv layer with kt = 4, T_out = 1, + LeakyReLU
//   outconv                             ReflectionPad2d(3) + 7x7 conv (first 3 outputs) + mean, centred crop  (CUDA cores)
// The gates need the mean of each conv output over (T, H, W): a separate reduction kernel (chan_sums) reads it back.
#include <cuda_fp16.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <cstring>
#include <functional>
#include <string>

#include "../../include/vfi_b200.h"
#include "vfi_internal.h"

namespace vfi {

namespace {

constexpr int kT = 4;  // planes per window (NBR_FRAME, flavr/__init__.py:12)
// conv layer ids (vfi_flavr_debug_conv / vfi_flavr_layer_plan)
constexpr int kEnc = 0;     // 10 * layer + 3 * block + {0 conv1, 1 conv2, 2 downsample}, layer 0..3
constexpr int kDec = 40;    // 40 + 4 * d + phase (py * 2 + px; phase 0 only for decoder 0 and 3)
constexpr int kFuse = 60;
constexpr int kNumLayers = 61;
const int kEncC[4] = {64, 128, 256, 512};

struct FBuf {
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

struct Gate {
  float* w = nullptr;  // [C][C]
  float* b = nullptr;  // [C]
  int C = 0;
};

}  // namespace

struct FlavrState : ModelState {
  int op_type = OP_F16;
  bool loaded = false;
  bool use_ref = false;  // debug: every conv through the CUDA-core checker
  int n_outputs = 1;
  bool enc_bias = false;
  std::vector<void*> allocs;
  float* stem_w = nullptr;  // [64][3][3][7][7]
  float* stem_b = nullptr;  // [64] (zeros without encoder bias)
  StreamConvLayer conv[kNumLayers];
  Gate enc_gate[4][2];
  Gate dec_gate[5];
  float* out_w = nullptr;  // outconv.1.weight[:3] [3][64][7][7]
  float* out_b = nullptr;
  // ---- workspace
  FBuf sums, xin, partial, gates;
  FBuf x0, x1, x2, x3, x4, xa, ta, tb, tr, s2d, ph, dxa, dxb, dxo, fz;
  ~FlavrState() override {
    for (void* p : allocs) cudaFree(p);
    for (FBuf* b : {&sums, &xin, &partial, &gates, &x0, &x1, &x2, &x3, &x4, &xa, &ta, &tb, &tr, &s2d, &ph, &dxa, &dxb, &dxo, &fz})
      b->release();
  }
};

namespace {

FlavrState* state(vfi_ctx* c) { return c ? static_cast<FlavrState*>(ctx_flavr(c)) : nullptr; }

#define XCK(call)                                                            \
  do {                                                                       \
    cudaError_t _e = (call);                                                 \
    if (_e != cudaSuccess) {                                                 \
      set_error(std::string(#call) + ": " + cudaGetErrorString(_e));         \
      return VFI_E_CUDA;                                                     \
    }                                                                        \
  } while (0)

#define XRUN(expr)           \
  do {                       \
    const int _rc = (expr);  \
    if (_rc) return _rc;     \
  } while (0)

int xfail(int code, const std::string& msg) {
  set_error(msg);
  return code;
}

template <class T>
int xupload(FlavrState* f, const T* h, size_t n, void** dptr) {
  void* d = nullptr;
  XCK(cudaMalloc(&d, n * sizeof(T)));
  f->allocs.push_back(d);
  XCK(cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice));
  *dptr = d;
  return VFI_OK;
}

// Packs one streamconv layer from wfun(n, dt, tap, padded input channel) and uploads it with its bias (nullptr: zeros).
int build_layer(FlavrState* f, StreamConvLayer& L, const std::function<float(int, int, int, int)>& wfun, const float* bias,
                int cout) {
  StreamConvParams p{};
  std::vector<uint16_t> pk;
  if (!pack_streamconv3d(L, f->op_type, wfun, &pk, &p)) return xfail(VFI_E_INVALID, "flavr: layer shape not supported by streamconv");
  std::vector<float> sh(L.n_total, 0.f);
  if (bias)
    for (int n = 0; n < cout; ++n) sh[n] = bias[n];
  void* d = nullptr;
  XRUN(xupload(f, pk.data(), pk.size(), &d));
  L.w = d;
  XRUN(xupload(f, sh.data(), sh.size(), &d));
  L.shift = static_cast<float*>(d);
  return VFI_OK;
}

StreamConvLayer layer3d(int ksize, int c0, int c1, int n, int kt, int pad_t, int T_out) {
  StreamConvLayer L;
  L.ksize = ksize;
  L.c0 = c0;
  L.c1 = c1;
  L.n_total = n;
  L.act = 0;
  L.kt = kt;
  L.pad_t = pad_t;
  L.T_in = kT;
  L.T_out = T_out;
  return L;
}

// Conv3d(cin, cout, 3, padding 1) weight [cout][cin][3][3][3] on cat(source 0, source 1)
int build_conv333(FlavrState* f, StreamConvLayer& L, int c0, int c1, int cout, const float* w, const float* bias) {
  L = layer3d(3, c0, c1, cout, 3, 1, kT);
  const int cin = c0 + c1;
  return build_layer(f, L, [&](int n, int dt, int tap, int j) { return w[(((size_t)n * cin + j) * 3 + dt) * 9 + tap]; },
                     bias, cout);
}

// Conv3d(cin, cout, 3, stride (1,2,2), padding 1) as a 2x2(x3) conv over the space-to-depth input [4 phases x cin]:
// phase (py, px) at channel (py * 2 + px) * cin; tap d (0 / 1) of an axis reads offset d - 1, i.e. kernel index
// 0 (d = 0, phase 1), 1 (d = 1, phase 0), 2 (d = 1, phase 1)
int build_conv_s2(FlavrState* f, StreamConvLayer& L, int cin, int cout, const float* w, const float* bias) {
  L = layer3d(2, 4 * cin, 0, cout, 3, 1, kT);
  L.pad_before = 1;
  return build_layer(f, L, [&](int n, int dt, int tap, int j) -> float {
    const int q = j / cin, c = j - q * cin, py = q >> 1, px = q & 1, dy = tap >> 1, dx = tap & 1;
    const int ky = dy == 0 ? (py ? 0 : -1) : 1 + py, kx = dx == 0 ? (px ? 0 : -1) : 1 + px;
    if (ky < 0 || kx < 0) return 0.f;
    return w[(((size_t)n * cin + c) * 3 + dt) * 9 + ky * 3 + kx];
  }, bias, cout);
}

// 1x1x1 downsample [cout][cin] (no bias); stride (1,2,2) reads the phase-(0,0) slice of the space-to-depth copy
int build_conv111(FlavrState* f, StreamConvLayer& L, int cin, int cout, const float* w) {
  L = layer3d(1, cin, 0, cout, 1, 0, kT);
  return build_layer(f, L, [&](int n, int, int, int j) { return w[(size_t)n * cin + j]; }, nullptr, cout);
}

// ConvTranspose3d(cin, cout, (3,4,4), stride (1,2,2), padding 1) weight [cin][cout][3][4][4]: output row 2 i + py sums
// input rows i + d - (1 - py), d = 0, 1, with kernel row 3 - py - 2 d; output plane t sums input planes t + dt - 1 with
// kernel plane 2 - dt.  Phase (py, px) = a 2x2(x3) conv with (1 - py, 1 - px) padding rows / columns before.
int build_convT_phase(FlavrState* f, StreamConvLayer& L, int c0, int c1, int cout, int py, int px, const float* w,
                      const float* bias) {
  L = layer3d(2, c0, c1, cout, 3, 1, kT);
  L.pad_before = 1 - py;
  L.pad_before_x = 1 - px;
  return build_layer(f, L, [&](int n, int dt, int tap, int j) -> float {
    const int ky = 3 - py - 2 * (tap >> 1), kx = 3 - px - 2 * (tap & 1);
    return w[((((size_t)j * cout + n) * 3 + (2 - dt)) * 4 + ky) * 4 + kx];
  }, bias, cout);
}

int build_gate(FlavrState* f, Gate& g, int C, const float* w, const float* b) {
  g.C = C;
  void* d = nullptr;
  XRUN(xupload(f, w, (size_t)C * C, &d));
  g.w = (float*)d;
  XRUN(xupload(f, b, (size_t)C, &d));
  g.b = (float*)d;
  return VFI_OK;
}

uint8_t* bp(const FBuf& b) { return static_cast<uint8_t*>(b.p); }

struct Runner {
  vfi_ctx* c;
  FlavrState* f;
  CtxInfo ci;
  cudaStream_t st;
  int S;  // windows of this pass
  int launches = 0;
  int ck(cudaError_t e, const char* what) {
    ++launches;
    if (e != cudaSuccess) {
      set_error(std::string("flavr: ") + what + ": " + cudaGetErrorString(e) + " / " + vfi_last_error());
      return VFI_E_CUDA;
    }
    return VFI_OK;
  }
  int conv(int id, const void* s0, int p0, const void* s1, int p1, void* out, int op, int H, int W) {
    return ck(launch_streamconv(f->conv[id], f->op_type, s0, p0, s1, p1, out, op, S, H, W, ci.num_sms, f->use_ref, st),
              "streamconv");
  }
  // the gate of a conv output x ([S*4][h][w][groups*C]); g <- sigmoid(W mean + b)
  int gate(const Gate& g, const void* x, int groups, int h, int w) {
    const size_t npx = (size_t)kT * h * w;
    XRUN(ck(launch_flavr_chan_sums(f->op_type, x, groups * g.C, npx, S, (float*)f->partial.p, st), "chan_sums"));
    return ck(launch_flavr_gate((const float*)f->partial.p, npx, groups, g.C, npx * groups, g.w, g.b, S, (float*)f->gates.p, st),
              "gate");
  }
  int apply(const void* x, int phases, const void* res, int act, void* out, void* s2d, int C, int H, int W) {
    return ck(launch_flavr_apply(f->op_type, x, phases, (const float*)f->gates.p, res, act, out, s2d, C, S * kT, kT, H, W, st),
              "apply");
  }
};

int ensure_workspace(FlavrState* f, int S, int Hp, int Wp) {
  const size_t P = (size_t)S * kT * (Hp / 2) * (Wp / 2);  // pixels of one plane set at H2
  const size_t e = 2;                                     // 16-bit
  XCK(f->sums.ensure((size_t)S * kT * 3 * 4));
  XCK(f->xin.ensure((size_t)S * kT * Hp * Wp * 16));
  XCK(f->partial.ensure((size_t)S * flavr_sum_chunks(P / S) * 512 * 4));
  XCK(f->gates.ensure((size_t)S * 512 * 4));
  for (FBuf* b : {&f->x0, &f->x1, &f->xa, &f->ta, &f->tb, &f->s2d, &f->dxa, &f->dxb}) XCK(b->ensure(64 * P * e));
  XCK(f->x2.ensure(32 * P * e));
  XCK(f->x3.ensure(16 * P * e));
  XCK(f->x4.ensure(32 * P * e));
  XCK(f->tr.ensure(32 * P * e));
  XCK(f->ph.ensure(256 * P * e));
  XCK(f->dxo.ensure(256 * P * e));
  XCK(f->fz.ensure(64 * P * e));
  return VFI_OK;
}

// replicate padding to a multiple of 16, centred (InputPadder, flavr_arch.py:200-206)
void pad16(int H, int W, int* Hp, int* Wp, int* pt, int* pl) {
  const int ph = ((H / 16) + 1) * 16 - H, pw = ((W / 16) + 1) * 16 - W;
  *Hp = H + ph % 16;
  *Wp = W + pw % 16;
  *pt = (ph % 16) / 2;
  *pl = (pw % 16) / 2;
}

int forward(vfi_ctx* c, FlavrState* f, const float* frames, int n_frames, int H, int W, int C, const int32_t* first, int S,
            float* out, cudaStream_t st) {
  int Hp, Wp, pt, pl;
  pad16(H, W, &Hp, &Wp, &pt, &pl);
  XRUN(ensure_workspace(f, S, Hp, Wp));
  Runner r{c, f, ctx_info(c), st, S};
  const int op = f->op_type;
  const int nimg = S * kT;
  const int H2 = Hp / 2, W2 = Wp / 2, H4 = Hp / 4, W4 = Wp / 4, H8 = Hp / 8, W8 = Wp / 8;
  FlavrFrameIdx idx{};
  for (int k = 0; k < S; ++k) {
    if (first[k] < 0 || first[k] + kT > n_frames) return xfail(VFI_E_INVALID, "flavr: window frame index out of range");
    for (int t = 0; t < kT; ++t) idx.i[k * kT + t] = first[k] + t;
  }
  // ---- normalisation and stem (UNet_3D_3D.forward :168-172, BasicStem)
  XRUN(r.ck(launch_flavr_frame_sums(frames, C, idx, nimg, H, W, Hp, Wp, pt, pl, (float*)f->sums.p, st), "frame_sums"));
  XRUN(r.ck(launch_flavr_prep(frames, C, idx, nimg, kT, H, W, Hp, Wp, pt, pl, (const float*)f->sums.p, (float4*)f->xin.p, st),
            "prep"));
  XRUN(r.ck(launch_flavr_stem(op, (const float4*)f->xin.p, nimg, kT, Hp, Wp, f->stem_w, f->stem_b, f->x0.p, st), "stem"));

  // ---- encoder (VideoResNet layer1..4, BasicBlock.forward)
  const int Hl[4] = {H2, H4, H8, H8}, Wl[4] = {W2, W4, W8, W8};
  const void* cur = f->x0.p;  // input of the next block, channel count cur_c
  int cur_c = 64;
  void* const skip_out[4] = {f->x1.p, f->x2.p, f->x3.p, f->x4.p};
  for (int l = 0; l < 4; ++l) {
    const int Co = kEncC[l], h = Hl[l], w = Wl[l];
    for (int b = 0; b < 2; ++b) {
      const int id = kEnc + 10 * l + 3 * b;
      const bool s2 = (l == 1 || l == 2) && b == 0;  // stride (1,2,2): read the space-to-depth copy of `cur`
      const void* res = cur;
      if (s2) {
        XRUN(r.conv(id, f->s2d.p, 4 * cur_c, nullptr, 0, f->ta.p, Co, h, w));
        XRUN(r.conv(id + 2, f->s2d.p, 4 * cur_c, nullptr, 0, f->tr.p, Co, h, w));
        res = f->tr.p;
      } else {
        XRUN(r.conv(id, cur, cur_c, nullptr, 0, f->ta.p, Co, h, w));
        if (f->conv[id + 2].w) {  // layer4 block 0: 256 -> 512 at stride 1
          XRUN(r.conv(id + 2, cur, cur_c, nullptr, 0, f->tr.p, Co, h, w));
          res = f->tr.p;
        }
      }
      XRUN(r.conv(id + 1, f->ta.p, Co, nullptr, 0, f->tb.p, Co, h, w));
      XRUN(r.gate(f->enc_gate[l][b], f->tb.p, 1, h, w));
      void* o = b == 0 ? f->xa.p : skip_out[l];
      void* s2d = (b == 1 && (l == 0 || l == 1)) ? f->s2d.p : nullptr;  // layer2 / layer3 read it
      XRUN(r.apply(f->tb.p, 0, res, 1, o, s2d, Co, h, w));
      cur = o;
      cur_c = Co;
    }
  }

  // ---- decoder (UNet_3D_3D.forward :176-189)
  // d = 0: conv(x4) -> dx3 (256 @ H8); 1: convT(dx3 | x3) -> dx2 (128 @ H4); 2: convT(dx2 | x2) -> dx1 (64 @ H2);
  // 3: conv(dx1 | x1) -> dx0 (64 @ H2); 4: convT(dx0 | x0) -> dx_out (64 @ Hp)
  struct Dec {
    const void* s0;
    int c0;
    const void* s1;
    int c1;
    int Co, h, w;  // output channels and the grid the conv runs on
    bool transposed;
    void* out;
  };
  const Dec dec[5] = {
      {f->x4.p, 512, nullptr, 0, 256, H8, W8, false, f->dxa.p},
      {f->dxa.p, 256, f->x3.p, 256, 128, H8, W8, true, f->dxb.p},
      {f->dxb.p, 128, f->x2.p, 128, 64, H4, W4, true, f->dxa.p},
      {f->dxa.p, 64, f->x1.p, 64, 64, H2, W2, false, f->dxb.p},
      {f->dxb.p, 64, f->x0.p, 64, 64, H2, W2, true, f->dxo.p},
  };
  for (int d = 0; d < 5; ++d) {
    const Dec& D = dec[d];
    if (D.transposed) {
      for (int q = 0; q < 4; ++q)
        XRUN(r.conv(kDec + 4 * d + q, D.s0, D.c0, D.s1, D.c1, bp(f->ph) + (size_t)q * D.Co * 2, 4 * D.Co, D.h, D.w));
      XRUN(r.gate(f->dec_gate[d], f->ph.p, 4, D.h, D.w));
      XRUN(r.apply(f->ph.p, 1, nullptr, 2, D.out, nullptr, D.Co, 2 * D.h, 2 * D.w));
    } else {
      XRUN(r.conv(kDec + 4 * d, D.s0, D.c0, D.s1, D.c1, f->tb.p, D.Co, D.h, D.w));
      XRUN(r.gate(f->dec_gate[d], f->tb.p, 1, D.h, D.w));
      XRUN(r.apply(f->tb.p, 0, nullptr, 2, D.out, nullptr, D.Co, D.h, D.w));
    }
  }
  // ---- feature_fuse over the four planes, LeakyReLU; outconv + mean, crop
  XRUN(r.conv(kFuse, f->dxo.p, 64, nullptr, 0, f->fz.p, 64, Hp, Wp));
  XRUN(r.ck(launch_flavr_outconv(op, f->fz.p, S, Hp, Wp, H, W, pt, pl, f->out_w, f->out_b, (const float*)f->sums.p, kT, out,
                                 st),
            "outconv"));
  ctx_add_launches(c, r.launches);
  return VFI_OK;
}

}  // namespace
}  // namespace vfi

using namespace vfi;

extern "C" {

/* tensor order: flavr_state_dict_names() in engine.py (UNet_3D_3D.state_dict() order) */
int vfi_flavr_load(vfi_ctx* c, const float* const* T, const int64_t* numel, int n_tensors, int operand_type) {
  if (!c || !T || !numel) return xfail(VFI_E_INVALID, "null argument");
  if (n_tensors != VFI_FLAVR_NUM_TENSORS && n_tensors != VFI_FLAVR_NUM_TENSORS_BIAS)
    return xfail(VFI_E_INVALID, "flavr: expected 59 (no encoder bias) or 76 tensors");
  if (operand_type != VFI_OPERAND_F16 && operand_type != VFI_OPERAND_BF16) return xfail(VFI_E_INVALID, "operand type");
  const CtxInfo ci = ctx_info(c);
  XCK(cudaSetDevice(ci.device));
  delete ctx_flavr(c);
  FlavrState* f = new FlavrState();
  ctx_flavr(c) = f;
  f->op_type = operand_type;
  f->enc_bias = n_tensors == VFI_FLAVR_NUM_TENSORS_BIAS;
  const bool eb = f->enc_bias;
  int t = 0;
  bool sizes_ok = true;
  auto take = [&](int64_t n) -> const float* {
    if (t >= n_tensors || numel[t] != n) sizes_ok = false;
    return sizes_ok ? T[t++] : nullptr;
  };
  void* d = nullptr;
  // ---- encoder.stem.0
  const float* sw = take(64LL * 3 * 3 * 49);
  std::vector<float> zeros(512, 0.f);
  const float* sb = eb ? take(64) : zeros.data();
  if (!sizes_ok) return xfail(VFI_E_INVALID, "flavr: stem tensor sizes");
  XRUN(xupload(f, sw, (size_t)64 * 441, &d));
  f->stem_w = (float*)d;
  XRUN(xupload(f, sb, 64, &d));
  f->stem_b = (float*)d;
  // ---- encoder.layer{1..4}.{0,1}: conv1.0, conv2.0, fg.attn_layer.0, downsample.0
  int cin = 64;
  for (int l = 0; l < 4; ++l) {
    const int Co = kEncC[l];
    for (int b = 0; b < 2; ++b) {
      const int ci = b == 0 ? cin : Co, id = kEnc + 10 * l + 3 * b;
      const bool s2 = (l == 1 || l == 2) && b == 0;
      const float* w1 = take((int64_t)Co * ci * 27);
      const float* b1 = eb ? take(Co) : nullptr;
      const float* w2 = take((int64_t)Co * Co * 27);
      const float* b2 = eb ? take(Co) : nullptr;
      const float* gw = take((int64_t)Co * Co);
      const float* gb = take(Co);
      const float* dw = (b == 0 && l > 0) ? take((int64_t)Co * ci) : nullptr;
      if (!sizes_ok) return xfail(VFI_E_INVALID, "flavr: encoder tensor sizes (layer " + std::to_string(l + 1) + ")");
      if (s2)
        XRUN(build_conv_s2(f, f->conv[id], ci, Co, w1, b1));
      else
        XRUN(build_conv333(f, f->conv[id], ci, 0, Co, w1, b1));
      f->conv[id].ext = 1;  // ReLU (PReLU with slope 0) in the epilogue
      f->conv[id].slope = 0.f;
      XRUN(build_conv333(f, f->conv[id + 1], Co, 0, Co, w2, b2));
      XRUN(build_gate(f, f->enc_gate[l][b], Co, gw, gb));
      if (dw) XRUN(build_conv111(f, f->conv[id + 2], ci, Co, dw));
    }
    cin = Co;
  }
  // ---- decoder.{0..4}: conv / upconv .0 weight + bias, then the gate (.1.attn_layer.0)
  const int dc0[5] = {512, 256, 128, 64, 64}, dc1[5] = {0, 256, 128, 64, 64}, dco[5] = {256, 128, 64, 64, 64};
  const bool dT[5] = {false, true, true, false, true};
  for (int k = 0; k < 5; ++k) {
    const int ci = dc0[k] + dc1[k], Co = dco[k];
    const float* w = take(dT[k] ? (int64_t)ci * Co * 48 : (int64_t)Co * ci * 27);
    const float* b = take(Co);
    const float* gw = take((int64_t)Co * Co);
    const float* gb = take(Co);
    if (!sizes_ok) return xfail(VFI_E_INVALID, "flavr: decoder tensor sizes (decoder." + std::to_string(k) + ")");
    if (dT[k]) {
      for (int q = 0; q < 4; ++q) XRUN(build_convT_phase(f, f->conv[kDec + 4 * k + q], dc0[k], dc1[k], Co, q >> 1, q & 1, w, b));
    } else {
      XRUN(build_conv333(f, f->conv[kDec + 4 * k], dc0[k], dc1[k], Co, w, b));
    }
    XRUN(build_gate(f, f->dec_gate[k], Co, gw, gb));
  }
  // ---- feature_fuse.conv.0 (64 x 256, no bias): temporal tap dt reads plane dt = input channels dt * 64 ..
  const float* fw = take(64LL * 256);
  if (!sizes_ok) return xfail(VFI_E_INVALID, "flavr: feature_fuse tensor size");
  {
    StreamConvLayer& L = f->conv[kFuse];
    L = layer3d(1, 64, 0, 64, kT, 0, 1);
    L.act = 1;
    XRUN(build_layer(f, L, [&](int n, int dt, int, int j) { return fw[(size_t)n * 256 + dt * 64 + j]; }, nullptr, 64));
  }
  // ---- outconv.1: [3 n_outputs][64][7][7]; only output 0 (channels 0..2) is used by the node
  if (t + 2 != n_tensors || numel[t] % (3 * 64 * 49) || numel[t] < 3 * 64 * 49 || numel[t + 1] * 64 * 49 != numel[t])
    return xfail(VFI_E_INVALID, "flavr: outconv tensor sizes");
  f->n_outputs = (int)(numel[t] / (3 * 64 * 49));
  XRUN(xupload(f, T[t], (size_t)3 * 64 * 49, &d));
  f->out_w = (float*)d;
  XRUN(xupload(f, T[t + 1], 3, &d));
  f->out_b = (float*)d;
  f->loaded = true;
  return VFI_OK;
}

int vfi_flavr_forward(vfi_ctx* c, const float* frames, int n_frames, int H, int W, int C, const int32_t* first_frame,
                      int n_windows, float* out, void* stream) {
  if (!c || !frames || !first_frame || !out) return xfail(VFI_E_INVALID, "null argument");
  FlavrState* f = state(c);
  if (!f || !f->loaded) return xfail(VFI_E_STATE, "vfi_flavr_load has not been called");
  if (n_windows < 1 || n_windows > VFI_FLAVR_MAX_WINDOWS) return xfail(VFI_E_INVALID, "flavr: n_windows must be in [1,8]");
  if (C < 3) return xfail(VFI_E_INVALID, "flavr: frames need >= 3 channels");
  if (H < 1 || W < 1) return xfail(VFI_E_INVALID, "flavr: empty frames");
  XCK(cudaSetDevice(ctx_info(c).device));
  return forward(c, f, frames, n_frames, H, W, C, first_frame, n_windows, out, static_cast<cudaStream_t>(stream));
}

int vfi_flavr_debug_set_ref(vfi_ctx* c, int use_ref) {
  FlavrState* f = state(c);
  if (!f) return xfail(VFI_E_STATE, "vfi_flavr_load has not been called");
  f->use_ref = use_ref != 0;
  return VFI_OK;
}

static const StreamConvLayer* flavr_layer(vfi_ctx* c, int layer) {
  FlavrState* f = state(c);
  if (!f || !f->loaded || layer < 0 || layer >= kNumLayers || !f->conv[layer].w) return nullptr;
  return &f->conv[layer];
}

int vfi_flavr_debug_conv(vfi_ctx* c, int layer, const void* src0, int pitch0, const void* src1, int pitch1, void* out,
                         int out_pitch, int n_windows, int H, int W, int impl, void* stream) {
  const StreamConvLayer* L = flavr_layer(c, layer);
  if (!L) return xfail(VFI_E_INVALID, "flavr: no such conv layer (or weights not loaded)");
  XCK(cudaSetDevice(ctx_info(c).device));
  const cudaError_t e = launch_streamconv(*L, state(c)->op_type, src0, pitch0, src1, pitch1, out, out_pitch, n_windows, H,
                                          W, ctx_info(c).num_sms, impl != 0, static_cast<cudaStream_t>(stream));
  ctx_add_launches(c, 1);
  if (e != cudaSuccess) return xfail(VFI_E_CUDA, std::string("streamconv: ") + cudaGetErrorString(e) + " / " + vfi_last_error());
  return VFI_OK;
}

int vfi_flavr_layer_plan(vfi_ctx* c, int layer, int32_t* info, int cap) {
  const StreamConvLayer* L = flavr_layer(c, layer);
  if (!L || !info) return xfail(VFI_E_INVALID, "flavr: no such conv layer (or weights not loaded)");
  StreamConvParams p{};
  if (!streamconv_plan(*L, &p)) return xfail(VFI_E_INVALID, "flavr: plan failed");
  const int32_t v[16] = {L->c0, L->c1, L->n_total, L->ksize, L->kt, L->pad_t, L->T_in, L->T_out, -p.halo_y0, -p.halo_x0,
                         p.n_cta, p.nsplit, p.a_slots, p.b_slots, (int32_t)p.smem_bytes, L->ext};
  for (int i = 0; i < cap && i < 16; ++i) info[i] = v[i];
  return VFI_OK;
}

int vfi_flavr_info(vfi_ctx* c, int* n_outputs, int* enc_bias) {
  FlavrState* f = state(c);
  if (!f || !f->loaded) return xfail(VFI_E_STATE, "vfi_flavr_load has not been called");
  if (n_outputs) *n_outputs = f->n_outputs;
  if (enc_bias) *enc_bias = f->enc_bias ? 1 : 0;
  return VFI_OK;
}

}  // extern "C"
