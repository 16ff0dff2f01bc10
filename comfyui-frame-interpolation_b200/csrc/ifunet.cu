// IFUNetModel on H100: weight packing (BatchNorm folded), the per-geometry workspace, the forward schedule and its C ABI
// (include/vfi_b200.h).  Reference: vfi_models/ifunet/IFUNet_arch.py, ifunet/__init__.py.
//
// Every convolution with 16 or more input channels is a streamconv layer; the CUDA-core stems and kernels around them
// are in ifunet_elem.cu.  Layer ids:
//   0 .. 9      FeatureNet UNetConv i (1..5), conv j: 2 (i - 1) + j.  conv1 (stride 2) runs as a 2x2 conv over the
//               space-to-depth copy (UNetConv 1: written by the level-input kernel), per-channel PReLU (ext 2)
//   10 + 6 u    UpConv u (0 deconv5, 1 deconv4, 2 deconv3): + 0..3 the ConvTranspose2d(4, 2, 1) phases (PReLU), + 4 conv1
//               on cat(up, skip) as two sources, + 5 conv2
//   28 + 8 b    IFBlock b: + 0..5 convblock (PReLU; + x as an element-wise add), + 6 flowconv (fp32 columns 0..3),
//               + 7 maskconvx{16, 8, 4} (1x1)
//   52          RRDBNet conv_first; 53 + 5 (3 r + d) + k: RRDB r, RDB d, conv k + 1 (conv1..4 LeakyReLU(0.2); conv5 ext 2
//               with slopes 1, the 0.2 folded into its weights and bias, the RDB input as residual); 143 conv_body (+
//               conv_first's output as residual), 144 conv_up1, 145 conv_up2, 146 conv_hr (LeakyReLU), 147 conv_last
//               (fp32 column 0)
//   148 + 12 b  ResynNet FlowBlock b: + 0 conv0.1, + 1 conv0.2 (stride 2; BatchNorm folded, PReLU), + 2..7 convblock,
//               + 8..11 lastconv phases (fp32 columns 0..3)
//   184, 185    context0.1, context1.1 (stride 2, PReLU); 186..189 decode.0 phases, 190..193 decode.1 phases (fp32)
//
// Channel layout.  A conv reads 64-channel k-blocks from at most two sources; padding channels meet zero weights and
// every conv writes its padding columns (zero weights, zero bias), so no channel a conv reads is ever stale:
//   FeatureNet levels        [C, pad to 64]; the space-to-depth copy: phase q at q * up8(C)
//   RDB (x, x1 .. x4)        x (64 channels) is source 0; x1 .. x4 live in one 128-channel growth tensor, 32 channels
//                            each at 0, 32, 64, 96, which is source 1: conv2 and conv3 read its first 64 channels, conv4
//                            and conv5 all 128 (conv2 and conv4 with zero weights on the slot not yet written).  The
//                            growth tensor is zeroed at the start of every call, so the unwritten slots hold zeros.
//   ConvT phases             [4][B][h][w][n] (phase q = py * 2 + px), interleaved by launch_ifunet_d2s
// Nearest x2 before conv_up1 and conv_up2 is materialized (launch_film_nearest16).
#include <cuda_fp16.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <string>

#include "../../include/vfi_b200.h"
#include "vfi_internal.h"

namespace vfi {

namespace {

constexpr int kBlk = 28, kFus = 52, kRes = 148, kCtx = 184, kDec = 186;
constexpr int kNumLayers = 194;
const int kFC[5] = {32, 64, 128, 256, 512};  // FeatureNet UNetConv 1..5 outputs
const int kBC[3] = {256, 128, 64};           // IFBlock channels
const int kBL[3] = {16, 8, 4};               // IFBlock levels (convex upsampling factor)

int up64(int v) { return (v + 63) / 64 * 64; }
int up8(int v) { return (v + 7) / 8 * 8; }

using Map = std::vector<int>;  // physical channel -> logical channel (-1: padding)
Map map_plain(int C, int P = -1) {
  Map m(P < 0 ? up64(C) : P);
  for (int j = 0; j < (int)m.size(); ++j) m[j] = j < C ? j : -1;
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
// RDB conv k (1..5): x at [0, 64), the growth tensor's slots at 64 + 32 s; conv k reads slots s < k - 1
Map map_rdb(int k) {
  Map m(k == 1 ? 64 : (k <= 3 ? 128 : 192), -1);
  for (int j = 0; j < (int)m.size(); ++j) m[j] = (j < 64 || (j - 64) / 32 < k - 1) ? j : -1;
  return m;
}

// ---------------------------------------------------------------- the state dict
struct Spec {
  std::vector<std::string> names;
  std::vector<int64_t> numel;
  void add(const std::string& n, int64_t v) {
    names.push_back(n);
    numel.push_back(v);
  }
  void conv_prelu(const std::string& p, int co, int ci, int k) {
    add(p + "0.weight", (int64_t)co * ci * k * k);
    add(p + "0.bias", co);
    add(p + "1.weight", co);
  }
  void bn(const std::string& p, int c) {
    for (const char* s : {"weight", "bias", "running_mean", "running_var"}) add(p + s, c);
    add(p + "num_batches_tracked", 1);
  }
  void cbam(const std::string& p, int c) {
    const int h = c / 16;
    add(p + "ChannelGate.mlp.1.weight", (int64_t)h * c);
    add(p + "ChannelGate.mlp.1.bias", h);
    add(p + "ChannelGate.mlp.3.weight", (int64_t)c * h);
    add(p + "ChannelGate.mlp.3.bias", c);
    add(p + "SpatialGate.spatial.conv.weight", 98);
    bn(p + "SpatialGate.spatial.bn.", 1);
  }
  void conv_bn(const std::string& p, int co, int ci) {
    add(p + "0.weight", (int64_t)co * ci * 9);
    bn(p + "1.", co);
    add(p + "2.weight", co);
  }
};

// IFUNetModel().state_dict() order (engine.py ifunet_state_dict_spec)
Spec make_spec() {
  Spec s;
  const std::string f = "flownet.fmap.";
  s.conv_prelu(f + "conv0.", 17, 7, 1);
  int cin = 17;
  for (int i = 0; i < 5; ++i) {
    const std::string p = f + "conv" + std::to_string(i + 1) + ".";
    s.conv_prelu(p + "conv1.", kFC[i], cin, 3);
    s.conv_prelu(p + "conv2.", kFC[i], kFC[i], 3);
    if (i > 0) s.cbam(p + "cbam.", kFC[i]);
    cin = kFC[i];
  }
  for (int u = 0; u < 3; ++u) {
    const int ci = 512 >> u, co = 256 >> u;
    const std::string p = f + "deconv" + std::to_string(5 - u) + ".";
    s.add(p + "deconv.0.weight", (int64_t)ci * (ci / 2) * 16);
    s.add(p + "deconv.0.bias", ci / 2);
    s.add(p + "deconv.1.weight", ci / 2);
    s.conv_prelu(p + "conv1.", ci / 2, ci, 3);
    s.conv_prelu(p + "conv2.", co, ci / 2, 3);
    if (u == 0) s.cbam(p + "cbam.", co);
  }
  for (int b = 0; b < 3; ++b) {
    const std::string p = "flownet.block" + std::to_string(b) + ".";
    const int c = kBC[b];
    for (int j = 0; j < 6; ++j) s.conv_prelu(p + "convblock." + std::to_string(j) + ".", c, c, 3);
    s.add(p + "flowconv.weight", (int64_t)4 * c * 9);
    s.add(p + "flowconv.bias", 4);
    for (int L : {16, 8, 4}) {
      s.add(p + "maskconvx" + std::to_string(L) + ".weight", (int64_t)L * L * 9 * c);
      s.add(p + "maskconvx" + std::to_string(L) + ".bias", L * L * 9);
    }
  }
  s.add("fusionnet.conv_first.weight", 64 * 16 * 9);
  s.add("fusionnet.conv_first.bias", 64);
  for (int r = 0; r < 6; ++r)
    for (int d = 1; d <= 3; ++d) {
      const std::string q = "fusionnet.body." + std::to_string(r) + ".rdb" + std::to_string(d) + ".";
      for (int k = 1; k <= 4; ++k) {
        s.add(q + "conv" + std::to_string(k) + ".weight", (int64_t)32 * (64 + 32 * (k - 1)) * 9);
        s.add(q + "conv" + std::to_string(k) + ".bias", 32);
      }
      s.add(q + "conv5.weight", 64 * 192 * 9);
      s.add(q + "conv5.bias", 64);
    }
  for (const char* n : {"conv_body", "conv_up1", "conv_up2", "conv_hr"}) {
    s.add(std::string("fusionnet.") + n + ".weight", 64 * 64 * 9);
    s.add(std::string("fusionnet.") + n + ".bias", 64);
  }
  s.add("fusionnet.conv_last.weight", 64 * 9);
  s.add("fusionnet.conv_last.bias", 1);
  for (int b = 0; b < 3; ++b) {
    const std::string p = "refinenet.block" + std::to_string(b) + ".";
    s.conv_bn(p + "conv0.0.", 64, b ? 12 : 6);
    s.conv_bn(p + "conv0.1.", 128, 64);
    s.conv_bn(p + "conv0.2.", 256, 128);
    for (int j = 0; j < 6; ++j) s.conv_bn(p + "convblock." + std::to_string(j) + ".", 256, 256);
    s.add(p + "lastconv.weight", 256 * 4 * 16);
    s.add(p + "lastconv.bias", 4);
  }
  s.conv_prelu("refinenet.degrad.conv0.", 32, 3, 3);
  for (int j = 1; j <= 3; ++j) s.conv_prelu("refinenet.degrad.conv" + std::to_string(j) + ".", 32, 32, 3);
  s.add("refinenet.degrad.deconv.1.weight", 128 * 32 * 16);
  s.add("refinenet.degrad.deconv.1.bias", 32);
  s.add("refinenet.degrad.deconv.2.weight", 32);
  s.add("refinenet.degrad.deconv.3.weight", 3 * 32 * 9);
  s.add("refinenet.degrad.deconv.3.bias", 3);
  for (int c = 0; c < 2; ++c) {
    s.conv_prelu("refinenet.context" + std::to_string(c) + ".0.", 16, 3, 3);
    s.conv_prelu("refinenet.context" + std::to_string(c) + ".1.", 32, 16, 3);
  }
  s.add("refinenet.decode.0.weight", 64 * 32 * 16);
  s.add("refinenet.decode.0.bias", 32);
  s.add("refinenet.decode.1.weight", 32 * 3 * 16);
  s.add("refinenet.decode.1.bias", 3);
  return s;
}

const Spec& spec() {
  static const Spec s = make_spec();
  return s;
}

struct IBuf {
  void* p = nullptr;
  size_t cap = 0;
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};

// ---------------------------------------------------------------- geometry
struct Geo {
  int H, W, Hp, Wp;
  double scale;
  int resize;                 // scale != 1: the flow net's inputs are resized, the IFBlock flows resized back
  int lh[6], lw[6];           // the flow net's input (floor(Hp * scale)) and its five stride-2 levels
  float cs_in, fs_in;         // F.interpolate(x, scale): coordinate scale (float)(1 / scale); flow multiplier (float) scale
  float cs_out, fm_out;       // F.interpolate(flow_up, 1 / scale) * (1 / scale)
};

int ifail(int code, const std::string& msg) {
  set_error(msg);
  return code;
}

std::string fmt_scale(double s) {
  char b[64];
  snprintf(b, sizeof b, "%g", s);
  return b;
}

// every size by the reference's arithmetic: F.interpolate(scale_factor=s) gives floor(n * s) (double), a stride-2
// conv ceil(n / 2), a ConvT 2 n; UpConv u's ConvT output must equal its skip (torch.cat), and each level's flow must
// come back to Hp x Wp (torch.cat with the frames at the next level, the flow sum, the fusion net's cat)
int geometry(int H, int W, double scale, Geo* g) {
  if (H < 1 || W < 1) return ifail(VFI_E_INVALID, "ifunet: empty frames");
  if (H > 16384 || W > 16384) return ifail(VFI_E_INVALID, "ifunet: frames larger than 16384 pixels on a side");
  if (!(scale > 0.0) || !std::isfinite(scale)) return ifail(VFI_E_INVALID, "ifunet: scale_factor must be a positive number");
  g->H = H;
  g->W = W;
  g->Hp = ((H - 1) / 64 + 1) * 64;
  g->Wp = ((W - 1) / 64 + 1) * 64;
  g->scale = scale;
  g->resize = scale != 1.0;
  const std::string what = "ifunet: the reference raises at scale_factor " + fmt_scale(scale) + " for a " +
                           std::to_string(H) + " x " + std::to_string(W) + " frame: ";
  const double h0 = g->resize ? std::floor((double)g->Hp * scale) : g->Hp;
  const double w0 = g->resize ? std::floor((double)g->Wp * scale) : g->Wp;
  if (h0 < 1.0 || w0 < 1.0) return ifail(VFI_E_INVALID, what + "the resized input is empty");
  if (h0 > 65536.0 || w0 > 65536.0) return ifail(VFI_E_INVALID, "ifunet: scale_factor " + fmt_scale(scale) + " is too large");
  g->lh[0] = (int)h0;
  g->lw[0] = (int)w0;
  for (int l = 1; l <= 5; ++l) {
    g->lh[l] = (g->lh[l - 1] + 1) / 2;
    g->lw[l] = (g->lw[l - 1] + 1) / 2;
  }
  const double inv = 1.0 / scale;
  for (int i = 0; i < 3; ++i) {
    for (int u = 4 - i; u <= 4; ++u)
      if (2 * g->lh[u + 1] != g->lh[u] || 2 * g->lw[u + 1] != g->lw[u])
        return ifail(VFI_E_INVALID, what + "a " + std::to_string(g->lh[u + 1]) + " x " + std::to_string(g->lw[u + 1]) +
                                        " UpConv input does not double to its " + std::to_string(g->lh[u]) + " x " +
                                        std::to_string(g->lw[u]) + " skip connection");
    const int L = kBL[i];
    const double fh = std::floor((double)(L * g->lh[4 - i]) * inv), fw = std::floor((double)(L * g->lw[4 - i]) * inv);
    if (fh != (double)g->Hp || fw != (double)g->Wp)
      return ifail(VFI_E_INVALID, what + "IFBlock " + std::to_string(i) + "'s flow comes back as " +
                                      std::to_string((long long)fh) + " x " + std::to_string((long long)fw) + ", not " +
                                      std::to_string(g->Hp) + " x " + std::to_string(g->Wp));
  }
  g->cs_in = (float)(1.0 / scale);
  g->fs_in = (float)scale;
  g->cs_out = (float)(1.0 / inv);
  g->fm_out = (float)inv;
  return VFI_OK;
}

// ---------------------------------------------------------------- workspace: one arena, a region per buffer
enum Buf : int {
  B_XIN, B_SK0, B_SK1, B_SK2, B_SK3, B_SK4, B_TMP, B_S2D, B_PH16, B_UP, B_Y1, B_Y2, B_XA, B_XB, B_FL16, B_FL32, B_MASK,
  B_UP32, B_FLOW, B_WARP, B_PSUM, B_PMAX, B_GATE, B_CMP,
  B_FIN, B_F0, B_X0, B_X1, B_X2, B_D, B_T, B_BIGA, B_BIGB, B_LAST, B_DEG,
  B_FBIN, B_RSTEM, B_RS2D, B_RC1, B_RC2, B_RA, B_RB, B_RPH16, B_RPH32, B_RFLOW, B_RMASK, B_RWARP,
  B_C0F, B_CAT, B_D0PH, B_D0, B_D1PH16, B_D1PH32, B_NUM
};

struct Layout {
  size_t off[B_NUM];
  size_t total;
};

Layout layout(const Geo& g) {
  size_t sz[B_NUM] = {0};
  const size_t e = 2, f4 = 4;
  auto px = [&](int l) { return (size_t)g.lh[l] * g.lw[l]; };
  const size_t F = (size_t)g.Hp * g.Wp, Q = F / 16, Hh = F / 4;
  sz[B_XIN] = 2 * px(1) * 128 * e;
  const Buf sk[5] = {B_SK0, B_SK1, B_SK2, B_SK3, B_SK4};
  size_t tmp = 0, s2d = 0, cmp = 0;
  for (int i = 0; i < 5; ++i) {
    sz[sk[i]] = 2 * px(i + 1) * up64(kFC[i]) * e;
    tmp = std::max(tmp, sz[sk[i]]);
    if (i > 0) s2d = std::max(s2d, 2 * px(i + 1) * map_s2d(kFC[i - 1]).size() * e);
    if (i > 0) cmp = std::max(cmp, 2 * px(i + 1) * 2 * f4);
  }
  sz[B_TMP] = tmp;
  size_t ph = 0, upc = 0;
  for (int u = 0; u < 3; ++u) {
    ph = std::max(ph, 4 * 2 * px(5 - u) * (size_t)(256 >> u) * e);
    upc = std::max(upc, 2 * px(4 - u) * (size_t)(256 >> u) * e);
  }
  sz[B_PH16] = ph;
  sz[B_UP] = sz[B_Y1] = sz[B_Y2] = upc;
  size_t xa = 0, fl16 = 0, fl32 = 0, mk = 0, up32 = 0;
  for (int b = 0; b < 3; ++b) {
    const size_t gp = px(4 - b);
    xa = std::max(xa, 2 * gp * kBC[b] * e);
    fl16 = std::max(fl16, 2 * gp * 16 * e);
    fl32 = std::max(fl32, 2 * gp * 4 * f4);
    mk = std::max(mk, 2 * gp * (size_t)(9 * kBL[b] * kBL[b]) * e);
    up32 = std::max(up32, 2 * gp * kBL[b] * kBL[b] * 4 * f4);
  }
  sz[B_XA] = sz[B_XB] = xa;
  sz[B_FL16] = fl16;
  sz[B_FL32] = fl32;
  sz[B_MASK] = mk;
  sz[B_UP32] = up32;
  sz[B_FLOW] = F * 4 * f4;
  sz[B_WARP] = F * 6 * f4;
  sz[B_PSUM] = sz[B_PMAX] = (size_t)2 * kIfuPoolChunks * 512 * f4;
  sz[B_GATE] = 2 * 512 * f4;
  sz[B_CMP] = cmp;
  sz[B_FIN] = sz[B_F0] = sz[B_X0] = sz[B_X1] = sz[B_X2] = sz[B_T] = Q * 64 * e;
  sz[B_D] = Q * 128 * e;
  sz[B_BIGA] = sz[B_BIGB] = F * 64 * e;
  sz[B_LAST] = F * 2 * f4;
  sz[B_DEG] = F * 3 * f4;
  sz[B_FBIN] = 2 * 12 * F * f4;
  sz[B_RSTEM] = 2 * Hh * 64 * e;
  sz[B_RS2D] = std::max(2 * Q * 256 * e, 2 * (F / 64) * 512 * e);
  sz[B_RC1] = 2 * Q * 128 * e;
  sz[B_RC2] = sz[B_RA] = sz[B_RB] = 2 * (F / 64) * 256 * e;
  sz[B_RPH16] = 4 * 2 * (F / 64) * 16 * e;
  sz[B_RPH32] = 4 * 2 * (F / 64) * 4 * f4;
  sz[B_RFLOW] = 2 * F * 2 * f4;
  sz[B_RMASK] = 2 * F * f4;
  sz[B_RWARP] = 2 * 3 * F * f4;
  sz[B_C0F] = 2 * Q * 32 * e;
  sz[B_CAT] = 2 * Q * 64 * e;
  sz[B_D0PH] = 4 * 2 * Q * 64 * e;
  sz[B_D0] = 2 * Hh * 64 * e;
  sz[B_D1PH16] = 4 * 2 * Hh * 16 * e;
  sz[B_D1PH32] = 4 * 2 * Hh * 4 * f4;
  Layout L{};
  size_t o = 0;
  for (int i = 0; i < B_NUM; ++i) {
    L.off[i] = o;
    o += (sz[i] + 255) / 256 * 256;
  }
  L.total = o;
  return L;
}

}  // namespace

struct IfunetState : ModelState {
  int op_type = OP_F16;
  bool loaded = false;
  bool use_ref = false;  // debug: every conv through the CUDA-core checker
  std::vector<void*> allocs;
  StreamConvLayer conv[kNumLayers];
  // CUDA-core weights: conv0 [17][7] + bias + slopes; CBAM k (FeatureNet conv2..5, deconv5): mlp, spatial [99];
  // FlowBlock stems [64][cin][9] + bias + slopes (BatchNorm folded); context stems [16][3][9] + bias + slopes
  float* c0[3] = {nullptr, nullptr, nullptr};
  float* cbam_mlp[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  float* cbam_sw[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  float* stem[3][3] = {};
  float* ctx[2][3] = {};
  IBuf arena;
  Layout lay{};
  ~IfunetState() override {
    for (void* p : allocs) cudaFree(p);
    arena.release();
  }
  uint8_t* at(Buf b) const { return static_cast<uint8_t*>(arena.p) + lay.off[b]; }
  float* f(Buf b) const { return reinterpret_cast<float*>(at(b)); }
};

namespace {

IfunetState* state(vfi_ctx* c) { return c ? static_cast<IfunetState*>(ctx_ifunet(c)) : nullptr; }

#define UCK(call)                                                            \
  do {                                                                       \
    cudaError_t _e = (call);                                                 \
    if (_e != cudaSuccess) {                                                 \
      set_error(std::string(#call) + ": " + cudaGetErrorString(_e));         \
      return VFI_E_CUDA;                                                     \
    }                                                                        \
  } while (0)

#define URUN(expr)           \
  do {                       \
    const int _rc = (expr);  \
    if (_rc) return _rc;     \
  } while (0)

template <class T>
int uupload(IfunetState* f, const T* h, size_t n, void** dptr) {
  void* d = nullptr;
  UCK(cudaMalloc(&d, n * sizeof(T)));
  f->allocs.push_back(d);
  UCK(cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice));
  *dptr = d;
  return VFI_OK;
}

int upload_f(IfunetState* f, const std::vector<float>& v, float** out) {
  void* d = nullptr;
  URUN(uupload(f, v.data(), v.size(), &d));
  *out = static_cast<float*>(d);
  return VFI_OK;
}

// the epilogue of a layer: ext 0 (act 0 / 1 = LeakyReLU(0.2)) or ext 2 (per-channel PReLU slopes; empty = identity,
// n_f32 fp32 columns)
struct Epi {
  int ext = 2, act = 0, n_f32 = 0;
};

// Packs one layer: input channels in_map (c0 from source 0, the rest from source 1), output columns out_map;
// wfun(logical output, tap, logical input), bias and slopes by logical output
int build_layer(IfunetState* f, StreamConvLayer& L, int ksize, const Map& in_map, int c0, const Map& out_map,
                const std::function<float(int, int, int)>& wfun, const std::vector<float>& bias,
                const std::vector<float>& slopes, Epi epi, int pad_y = -1, int pad_x = -1) {
  L = StreamConvLayer{};
  L.ksize = ksize;
  L.c0 = c0;
  L.c1 = (int)in_map.size() - c0;
  L.n_total = (int)out_map.size();
  L.act = epi.act;
  L.ext = epi.ext;
  L.n_f32 = epi.n_f32;
  L.pad_before = pad_y;
  L.pad_before_x = pad_x;
  std::vector<uint16_t> pk;
  StreamConvParams p{};
  if (!pack_streamconv(L, f->op_type, [&](int n, int tap, int j) -> float {
        const int lo = out_map[n], li = in_map[j];
        return (lo < 0 || li < 0) ? 0.f : wfun(lo, tap, li);
      }, &pk, &p))
    return ifail(VFI_E_INVALID, "ifunet: layer shape not supported by streamconv");
  std::vector<float> sh(L.n_total, 0.f), sl(L.n_total, 1.f);
  for (int n = 0; n < L.n_total; ++n) {
    const int lo = out_map[n];
    if (lo < 0) continue;
    sh[n] = bias[lo];
    if (!slopes.empty()) sl[n] = slopes[lo];
  }
  void* d = nullptr;
  URUN(uupload(f, pk.data(), pk.size(), &d));
  L.w = d;
  URUN(upload_f(f, sh, &L.shift));
  if (L.ext == 2) {
    float* s = nullptr;
    URUN(upload_f(f, sl, &s));
    L.slopes = s;
  }
  return VFI_OK;
}

std::vector<float> vec(const float* p, int n, float mul = 1.f) {
  std::vector<float> v(n);
  for (int i = 0; i < n; ++i) v[i] = p[i] * mul;
  return v;
}

// Conv2d(cin, cout, k, 1, k / 2) weight [cout][cin][k][k], each output row times oscale[lo] (empty: 1)
int build_conv(IfunetState* f, int id, int k, const Map& in, int c0, const Map& out, int cin, const float* w,
               const std::vector<float>& bias, const std::vector<float>& slopes, Epi epi,
               const std::vector<float>& oscale = {}) {
  return build_layer(f, f->conv[id], k, in, c0, out, [&](int lo, int tap, int li) {
    return w[((size_t)lo * cin + li) * k * k + tap] * (oscale.empty() ? 1.f : oscale[lo]);
  }, bias, slopes, epi);
}

// Conv2d(cin, cout, 3, stride 2, padding 1) as a 2x2 conv over the space-to-depth copy (logical input q * cin + c):
// tap d (0 / 1) of an axis reads offset d - 1, i.e. kernel index 0 (d = 0, phase 1), 1 (d = 1, phase 0), 2 (d = 1, phase 1)
int build_conv_s2(IfunetState* f, int id, int cin, const Map& out, const float* w, const std::vector<float>& bias,
                  const std::vector<float>& slopes, const std::vector<float>& oscale = {}) {
  const Map in = map_s2d(cin);
  return build_layer(f, f->conv[id], 2, in, (int)in.size(), out, [&](int lo, int tap, int li) -> float {
    const int q = li / cin, c = li - q * cin, py = q >> 1, px = q & 1, dy = tap >> 1, dx = tap & 1;
    const int ky = dy == 0 ? (py ? 0 : -1) : 1 + py, kx = dx == 0 ? (px ? 0 : -1) : 1 + px;
    if (ky < 0 || kx < 0) return 0.f;
    return w[((size_t)lo * cin + c) * 9 + ky * 3 + kx] * (oscale.empty() ? 1.f : oscale[lo]);
  }, bias, slopes, Epi{}, 1);
}

// ConvTranspose2d(cin, cout, 4, 2, 1) weight [cin][cout][4][4]: output row 2 i + py sums input rows i + d - (1 - py),
// d = 0, 1, with kernel row 3 - py - 2 d.  Phase q = (py, px): a 2x2 conv with (1 - py, 1 - px) padding before.
int build_convT(IfunetState* f, int id0, const Map& in, const Map& out, int cout, const float* w,
                const std::vector<float>& bias, const std::vector<float>& slopes, Epi epi) {
  for (int q = 0; q < 4; ++q) {
    const int py = q >> 1, px = q & 1;
    URUN(build_layer(f, f->conv[id0 + q], 2, in, (int)in.size(), out, [&](int lo, int tap, int li) {
      const int ky = 3 - py - 2 * (tap >> 1), kx = 3 - px - 2 * (tap & 1);
      return w[(((size_t)li * cout + lo) * 4 + ky) * 4 + kx];
    }, bias, slopes, epi, 1 - py, 1 - px));
  }
  return VFI_OK;
}

// eval-mode BatchNorm (eps 1e-5) as a per-channel scale and shift: y = x * scale + shift
void bn_fold(const float* g, const float* b, const float* mean, const float* var, int n, std::vector<float>* scale,
             std::vector<float>* shift) {
  scale->resize(n);
  shift->resize(n);
  for (int i = 0; i < n; ++i) {
    const double s = (double)g[i] / std::sqrt((double)var[i] + 1e-5);
    (*scale)[i] = (float)s;
    (*shift)[i] = (float)((double)b[i] - (double)mean[i] * s);
  }
}

struct Runner {
  IfunetState* f;
  CtxInfo ci;
  cudaStream_t st;
  int launches = 0;
  int ck(cudaError_t e, const char* what) {
    ++launches;
    if (e != cudaSuccess) {
      set_error(std::string("ifunet: ") + what + ": " + cudaGetErrorString(e) + " / " + vfi_last_error());
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

// FeatureNet (the level input is in B_XIN) for B images; the output (C = kBC[level]) in B_Y2
int fmap(Runner& r, const Geo& g, int level, int B) {
  IfunetState* f = r.f;
  const int op = f->op_type;
  const Buf sk[5] = {B_SK0, B_SK1, B_SK2, B_SK3, B_SK4};
  URUN(r.conv(0, f->at(B_XIN), 128, nullptr, 0, f->at(B_TMP), 64, B, g.lh[1], g.lw[1]));
  URUN(r.conv(1, f->at(B_TMP), 64, nullptr, 0, f->at(B_SK0), 64, B, g.lh[1], g.lw[1]));
  for (int i = 1; i < 5; ++i) {
    const int Pi = up64(kFC[i - 1]), Ps = (int)map_s2d(kFC[i - 1]).size(), Po = up64(kFC[i]);
    URUN(r.ck(launch_ifunet_s2d(op, f->at(sk[i - 1]), Pi, up8(kFC[i - 1]), B, g.lh[i], g.lw[i], f->at(B_S2D), Ps, r.st),
              "s2d"));
    URUN(r.conv(2 * i, f->at(B_S2D), Ps, nullptr, 0, f->at(B_TMP), Po, B, g.lh[i + 1], g.lw[i + 1]));
    URUN(r.conv(2 * i + 1, f->at(B_TMP), Po, nullptr, 0, f->at(sk[i]), Po, B, g.lh[i + 1], g.lw[i + 1]));
    URUN(r.ck(launch_ifunet_cbam(op, f->at(sk[i]), Po, kFC[i], B, g.lh[i + 1], g.lw[i + 1], f->cbam_mlp[i - 1],
                                 f->cbam_sw[i - 1], f->f(B_PSUM), f->f(B_PMAX), f->f(B_GATE), f->f(B_CMP), r.st),
              "cbam"));
  }
  const uint8_t* y = f->at(B_SK4);
  for (int u = 0; u <= level; ++u) {
    const int ci = 512 >> u, cp = ci / 2, co = 256 >> u, id = 10 + 6 * u;
    const int hs = g.lh[5 - u], ws = g.lw[5 - u], hb = g.lh[4 - u], wb = g.lw[4 - u];
    for (int q = 0; q < 4; ++q)
      URUN(r.conv(id + q, y, ci, nullptr, 0, f->at(B_PH16) + (size_t)q * B * hs * ws * cp * 2, cp, B, hs, ws));
    URUN(r.ck(launch_ifunet_d2s(f->at(B_PH16), cp, B, hs, ws, f->at(B_UP), r.st), "d2s"));
    URUN(r.conv(id + 4, f->at(B_UP), cp, f->at(sk[3 - u]), cp, f->at(B_Y1), cp, B, hb, wb));
    URUN(r.conv(id + 5, f->at(B_Y1), cp, nullptr, 0, f->at(B_Y2), co, B, hb, wb));
    if (u == 0)
      URUN(r.ck(launch_ifunet_cbam(op, f->at(B_Y2), co, co, B, hb, wb, f->cbam_mlp[4], f->cbam_sw[4], f->f(B_PSUM),
                                   f->f(B_PMAX), f->f(B_GATE), f->f(B_CMP), r.st),
                "cbam"));
    y = f->at(B_Y2);
  }
  return VFI_OK;
}

// IFBlock b on the FeatureNet output (B_Y2, B images), then the flow update of `mode` (launch_ifunet_flow_update)
int ifblock(Runner& r, const Geo& g, int b, int B, int mode) {
  IfunetState* f = r.f;
  const int op = f->op_type, C = kBC[b], L = kBL[b], gh = g.lh[4 - b], gw = g.lw[4 - b], id = kBlk + 8 * b;
  const uint8_t* src = f->at(B_Y2);
  for (int j = 0; j < 6; ++j) {
    uint8_t* dst = f->at(j % 2 ? B_XB : B_XA);
    URUN(r.conv(id + j, src, C, nullptr, 0, dst, C, B, gh, gw));
    src = dst;
  }
  URUN(r.ck(launch_ifunet_add16(op, f->at(B_XB), f->at(B_Y2), (size_t)B * gh * gw * C, r.st), "add16"));
  URUN(r.conv(id + 6, f->at(B_XB), C, nullptr, 0, f->at(B_FL16), 16, B, gh, gw, nullptr, f->f(B_FL32), 4));
  URUN(r.conv(id + 7, f->at(B_XB), C, nullptr, 0, f->at(B_MASK), 9 * L * L, B, gh, gw));
  URUN(r.ck(launch_ifunet_convex(op, f->f(B_FL32), f->at(B_MASK), L, B, gh, gw, f->f(B_UP32), r.st), "convex"));
  return r.ck(launch_ifunet_flow_update(f->f(B_UP32), L * gh, L * gw, g.resize, g.cs_out, g.fm_out, mode, g.Hp, g.Wp,
                                        f->f(B_FLOW), r.st),
              "flow_update");
}

IfuFlowIn flow_in_args(const IfunetState* f, const Geo& g, const float* img0, const float* img1, int level, int swap0,
                       float t) {
  IfuFlowIn a{};
  a.f0 = img0;
  a.f1 = img1;
  a.H = g.H;
  a.W = g.W;
  a.Hp = g.Hp;
  a.Wp = g.Wp;
  a.warped = level ? f->f(B_WARP) : nullptr;
  a.flow = level ? f->f(B_FLOW) : nullptr;
  a.swap0 = swap0;
  a.t = t;
  a.resize = g.resize;
  a.cscale = g.cs_in;
  a.fscale = g.fs_in;
  a.h0 = g.lh[0];
  a.w0 = g.lw[0];
  a.c0w = f->c0[0];
  a.c0b = f->c0[1];
  a.c0s = f->c0[2];
  return a;
}

// one RDB: x (64 channels) -> out (64 channels), the growth tensor B_D
int rdb(Runner& r, const Geo& g, int id, const void* x, void* out) {
  IfunetState* f = r.f;
  const int h = g.Hp / 4, w = g.Wp / 4;
  uint8_t* D = f->at(B_D);
  URUN(r.conv(id, x, 64, nullptr, 0, D, 128, 1, h, w));
  URUN(r.conv(id + 1, x, 64, D, 128, D + 32 * 2, 128, 1, h, w));
  URUN(r.conv(id + 2, x, 64, D, 128, D + 64 * 2, 128, 1, h, w));
  URUN(r.conv(id + 3, x, 64, D, 128, D + 96 * 2, 128, 1, h, w));
  return r.conv(id + 4, x, 64, D, 128, out, 64, 1, h, w, x);
}

int forward(vfi_ctx* c, IfunetState* f, const float* img0, const float* img1, const Geo& g, float t, bool ensemble,
            float* out, cudaStream_t st) {
  const int op = f->op_type;
  Runner r{f, ctx_info(c), st};
  const int Hp = g.Hp, Wp = g.Wp;
  // ---- IFUNet: three levels; level 0's ensemble pass is independent of the first, so both run as one batch
  for (int i = 0; i < 3; ++i) {
    const int passes = (i == 0 || !ensemble) ? 1 : 2;
    for (int k = 0; k < passes; ++k) {
      const int B = (i == 0 && ensemble) ? 2 : 1;
      const IfuFlowIn a = flow_in_args(f, g, img0, img1, i, k, t);
      URUN(r.ck(launch_ifunet_flow_in(op, a, B, f->at(B_XIN), st), "flow_in"));
      URUN(fmap(r, g, i, B));
      const int mode = i == 0 ? (ensemble ? 1 : 0) : (k == 0 ? 2 : 3);
      URUN(ifblock(r, g, i, B, mode));
    }
    URUN(r.ck(launch_ifunet_warp_frames(img0, img1, g.H, g.W, Hp, Wp, f->f(B_FLOW), f->f(B_WARP), st), "warp_frames"));
  }
  // ---- RRDBNet fusion at 1/4, the mask and merged = w0 * mask + w1 * (1 - mask)
  const int hq = Hp / 4, wq = Wp / 4;
  UCK(cudaMemsetAsync(f->at(B_D), 0, (size_t)hq * wq * 128 * 2, st));
  URUN(r.ck(launch_ifunet_fusion_in(op, img0, img1, g.H, g.W, Hp, Wp, f->f(B_WARP), f->f(B_FLOW), f->at(B_FIN), st),
            "fusion_in"));
  URUN(r.conv(kFus, f->at(B_FIN), 64, nullptr, 0, f->at(B_F0), 64, 1, hq, wq));
  Buf in = B_F0;
  for (int rr = 0; rr < 6; ++rr) {
    Buf fr[2];
    int n = 0;
    for (Buf b : {B_X0, B_X1, B_X2})
      if (b != in && n < 2) fr[n++] = b;
    const int id = kFus + 1 + 15 * rr;
    URUN(rdb(r, g, id, f->at(in), f->at(fr[0])));
    URUN(rdb(r, g, id + 5, f->at(fr[0]), f->at(fr[1])));
    URUN(rdb(r, g, id + 10, f->at(fr[1]), f->at(fr[0])));
    URUN(r.ck(launch_ifunet_rrdb_res(op, f->at(fr[0]), f->at(in), (size_t)hq * wq * 64, st), "rrdb_res"));
    in = fr[0];
  }
  URUN(r.conv(kFus + 91, f->at(in), 64, nullptr, 0, f->at(B_T), 64, 1, hq, wq, f->at(B_F0)));
  URUN(r.ck(launch_film_nearest16(f->at(B_T), hq, wq, f->at(B_BIGA), 64, 1, 2 * hq, 2 * wq, st), "nearest16"));
  URUN(r.conv(kFus + 92, f->at(B_BIGA), 64, nullptr, 0, f->at(B_BIGB), 64, 1, 2 * hq, 2 * wq));
  URUN(r.ck(launch_film_nearest16(f->at(B_BIGB), 2 * hq, 2 * wq, f->at(B_BIGA), 64, 1, Hp, Wp, st), "nearest16"));
  URUN(r.conv(kFus + 93, f->at(B_BIGA), 64, nullptr, 0, f->at(B_BIGB), 64, 1, Hp, Wp));
  URUN(r.conv(kFus + 94, f->at(B_BIGB), 64, nullptr, 0, f->at(B_BIGA), 64, 1, Hp, Wp));
  URUN(r.conv(kFus + 95, f->at(B_BIGA), 64, nullptr, 0, f->at(B_BIGB), 16, 1, Hp, Wp, nullptr, f->f(B_LAST), 2));
  URUN(r.ck(launch_ifunet_merge(f->f(B_WARP), f->f(B_LAST), Hp, Wp, f->f(B_DEG), st), "merge"));
  // ---- ResynNet: both frames as one batch of two
  const size_t F = (size_t)Hp * Wp;
  for (int b = 0; b < 3; ++b) {
    const int s = b == 0 ? 4 : (b == 1 ? 2 : 1), cin = b ? 12 : 6, id = kRes + 12 * b;
    const int h1 = Hp / s, w1 = Wp / s, h2 = h1 / 2, w2 = w1 / 2, h4 = h1 / 4, w4 = w1 / 4, h8 = h1 / 8, w8 = w1 / 8;
    URUN(r.ck(launch_ifunet_fb_in(img0, img1, g.H, g.W, Hp, Wp, f->f(B_DEG), f->f(B_RWARP), f->f(B_RMASK), f->f(B_RFLOW),
                                  cin, s, f->f(B_FBIN), st),
              "fb_in"));
    const float* fb = f->f(B_FBIN);
    URUN(r.ck(launch_ifunet_stem(op, fb, fb + (size_t)cin * h1 * w1, cin, h1, w1, h1, w1, f->stem[b][0], f->stem[b][1],
                                 f->stem[b][2], 64, 2, 64, f->at(B_RSTEM), st),
              "stem"));
    URUN(r.ck(launch_ifunet_s2d(op, f->at(B_RSTEM), 64, 64, 2, h2, w2, f->at(B_RS2D), 256, st), "s2d"));
    URUN(r.conv(id, f->at(B_RS2D), 256, nullptr, 0, f->at(B_RC1), 128, 2, h4, w4));
    URUN(r.ck(launch_ifunet_s2d(op, f->at(B_RC1), 128, 128, 2, h4, w4, f->at(B_RS2D), 512, st), "s2d"));
    URUN(r.conv(id + 1, f->at(B_RS2D), 512, nullptr, 0, f->at(B_RC2), 256, 2, h8, w8));
    const uint8_t* src = f->at(B_RC2);
    for (int j = 0; j < 6; ++j) {
      uint8_t* dst = f->at(j % 2 ? B_RB : B_RA);
      URUN(r.conv(id + 2 + j, src, 256, nullptr, 0, dst, 256, 2, h8, w8));
      src = dst;
    }
    URUN(r.ck(launch_ifunet_add16(op, f->at(B_RB), f->at(B_RC2), (size_t)2 * h8 * w8 * 256, st), "add16"));
    for (int q = 0; q < 4; ++q)
      URUN(r.conv(id + 8 + q, f->at(B_RB), 256, nullptr, 0, f->at(B_RPH16) + (size_t)q * 2 * h8 * w8 * 16 * 2, 16, 2, h8, w8,
                  nullptr, f->f(B_RPH32) + (size_t)q * 2 * h8 * w8 * 4, 4));
    URUN(r.ck(launch_ifunet_fb_out(f->f(B_RPH32), h8, w8, s, b == 0, img0, img1, g.H, g.W, Hp, Wp, f->f(B_RFLOW),
                                   f->f(B_RMASK), f->f(B_RWARP), st),
              "fb_out"));
  }
  // context0 on the frames, warped by the flow at 1/4; context1 on the warped frames; decode
  URUN(r.ck(launch_ifunet_stem(op, img0, img1, 3, Hp, Wp, g.H, g.W, f->ctx[0][0], f->ctx[0][1], f->ctx[0][2], 16, 2, 64,
                               f->at(B_RSTEM), st),
            "stem"));
  URUN(r.ck(launch_ifunet_s2d(op, f->at(B_RSTEM), 64, 16, 2, Hp / 2, Wp / 2, f->at(B_RS2D), 64, st), "s2d"));
  URUN(r.conv(kCtx, f->at(B_RS2D), 64, nullptr, 0, f->at(B_C0F), 32, 2, hq, wq));
  URUN(r.ck(launch_ifunet_ctx_warp(op, f->at(B_C0F), 32, f->f(B_RFLOW), Hp, Wp, f->at(B_CAT), st), "ctx_warp"));
  const float* rw = f->f(B_RWARP);
  URUN(r.ck(launch_ifunet_stem(op, rw, rw + 3 * F, 3, Hp, Wp, Hp, Wp, f->ctx[1][0], f->ctx[1][1], f->ctx[1][2], 16, 2, 64,
                               f->at(B_RSTEM), st),
            "stem"));
  URUN(r.ck(launch_ifunet_s2d(op, f->at(B_RSTEM), 64, 16, 2, Hp / 2, Wp / 2, f->at(B_RS2D), 64, st), "s2d"));
  URUN(r.conv(kCtx + 1, f->at(B_RS2D), 64, nullptr, 0, f->at(B_CAT) + 32 * 2, 64, 2, hq, wq));
  for (int q = 0; q < 4; ++q)
    URUN(r.conv(kDec + q, f->at(B_CAT), 64, nullptr, 0, f->at(B_D0PH) + (size_t)q * 2 * hq * wq * 64 * 2, 64, 2, hq, wq));
  URUN(r.ck(launch_ifunet_d2s(f->at(B_D0PH), 64, 2, hq, wq, f->at(B_D0), st), "d2s"));
  const size_t hh = (size_t)(Hp / 2) * (Wp / 2);
  for (int q = 0; q < 4; ++q)
    URUN(r.conv(kDec + 4 + q, f->at(B_D0), 64, nullptr, 0, f->at(B_D1PH16) + (size_t)q * 2 * hh * 16 * 2, 16, 2, Hp / 2,
                Wp / 2, nullptr, f->f(B_D1PH32) + (size_t)q * 2 * hh * 4, 4));
  URUN(r.ck(launch_ifunet_final(f->f(B_D1PH32), f->f(B_RWARP), f->f(B_RMASK), f->f(B_DEG), g.H, g.W, Hp, Wp, out, st),
            "final"));
  ctx_add_launches(c, r.launches);
  return VFI_OK;
}

// the arena for a geometry; a workspace the device cannot hold is refused before anything runs
int ensure_workspace(IfunetState* f, const Geo& g) {
  f->lay = layout(g);
  if (f->lay.total <= f->arena.cap) return VFI_OK;
  f->arena.release();
  size_t free_b = f->lay.total, total_b = 0;
#ifndef VFI_HOST_EMU
  UCK(cudaMemGetInfo(&free_b, &total_b));
#endif
  (void)total_b;
  if (f->lay.total > free_b)
    return ifail(VFI_E_INVALID, "ifunet: a " + std::to_string(g.H) + " x " + std::to_string(g.W) + " frame at scale_factor " +
                                    fmt_scale(g.scale) + " needs " + std::to_string(f->lay.total >> 20) +
                                    " MiB of workspace; the device has " + std::to_string(free_b >> 20) + " MiB free");
  void* p = nullptr;
  const cudaError_t e = cudaMalloc(&p, f->lay.total);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return ifail(VFI_E_INVALID, "ifunet: could not allocate " + std::to_string(f->lay.total >> 20) +
                                    " MiB of workspace: " + cudaGetErrorString(e));
  }
  f->arena.p = p;
  f->arena.cap = f->lay.total;
  return VFI_OK;
}

}  // namespace
}  // namespace vfi

using namespace vfi;

extern "C" {

/* tensor order: IFUNetModel().state_dict() (engine.py ifunet_state_dict_spec) */
int vfi_ifunet_load(vfi_ctx* c, const float* const* T, const int64_t* numel, int n_tensors, int operand_type) {
  if (!c || !T || !numel) return ifail(VFI_E_INVALID, "null argument");
  const Spec& sp = spec();
  if (n_tensors != (int)sp.names.size())
    return ifail(VFI_E_INVALID, "ifunet: expected " + std::to_string(sp.names.size()) + " tensors, got " +
                                    std::to_string(n_tensors));
  if (operand_type != VFI_OPERAND_F16 && operand_type != VFI_OPERAND_BF16) return ifail(VFI_E_INVALID, "operand type");
  std::map<std::string, const float*> by;
  for (int i = 0; i < n_tensors; ++i) {
    if (!T[i] || numel[i] != sp.numel[i])
      return ifail(VFI_E_INVALID, "ifunet: tensor " + std::to_string(i) + " (" + sp.names[i] + ") has " +
                                      std::to_string((long long)numel[i]) + " elements, IFUNetModel has " +
                                      std::to_string((long long)sp.numel[i]));
    by[sp.names[i]] = T[i];
  }
  auto W = [&](const std::string& n) { return by.at(n); };
  const CtxInfo ci = ctx_info(c);
  UCK(cudaSetDevice(ci.device));
  delete ctx_ifunet(c);
  IfunetState* f = new IfunetState();
  ctx_ifunet(c) = f;
  f->op_type = operand_type;
  const std::string fm = "flownet.fmap.";
  const std::vector<float> none;
  // ---- FeatureNet
  URUN(upload_f(f, vec(W(fm + "conv0.0.weight"), 17 * 7), &f->c0[0]));
  URUN(upload_f(f, vec(W(fm + "conv0.0.bias"), 17), &f->c0[1]));
  URUN(upload_f(f, vec(W(fm + "conv0.1.weight"), 17), &f->c0[2]));
  int cin = 17;
  for (int i = 0; i < 5; ++i) {
    const std::string p = fm + "conv" + std::to_string(i + 1) + ".";
    const int C = kFC[i];
    URUN(build_conv_s2(f, 2 * i, cin, map_plain(C), W(p + "conv1.0.weight"), vec(W(p + "conv1.0.bias"), C),
                       vec(W(p + "conv1.1.weight"), C)));
    URUN(build_conv(f, 2 * i + 1, 3, map_plain(C), up64(C), map_plain(C), C, W(p + "conv2.0.weight"),
                    vec(W(p + "conv2.0.bias"), C), vec(W(p + "conv2.1.weight"), C), Epi{}));
    cin = C;
  }
  auto load_cbam = [&](int k, const std::string& p, int C) -> int {
    const int h = C / 16;
    std::vector<float> mlp;
    for (auto [n, cnt] : {std::pair<const char*, int>{"ChannelGate.mlp.1.weight", h * C}, {"ChannelGate.mlp.1.bias", h},
                          {"ChannelGate.mlp.3.weight", C * h}, {"ChannelGate.mlp.3.bias", C}}) {
      const float* t = W(p + n);
      mlp.insert(mlp.end(), t, t + cnt);
    }
    std::vector<float> sc, shf;
    const std::string b = p + "SpatialGate.spatial.bn.";
    bn_fold(W(b + "weight"), W(b + "bias"), W(b + "running_mean"), W(b + "running_var"), 1, &sc, &shf);
    std::vector<float> sw = vec(W(p + "SpatialGate.spatial.conv.weight"), 98, sc[0]);
    sw.push_back(shf[0]);
    URUN(upload_f(f, mlp, &f->cbam_mlp[k]));
    return upload_f(f, sw, &f->cbam_sw[k]);
  };
  for (int i = 1; i < 5; ++i) URUN(load_cbam(i - 1, fm + "conv" + std::to_string(i + 1) + ".cbam.", kFC[i]));
  for (int u = 0; u < 3; ++u) {
    const int ci = 512 >> u, cp = ci / 2, co = 256 >> u, id = 10 + 6 * u;
    const std::string p = fm + "deconv" + std::to_string(5 - u) + ".";
    URUN(build_convT(f, id, map_plain(ci), map_plain(cp), cp, W(p + "deconv.0.weight"), vec(W(p + "deconv.0.bias"), cp),
                     vec(W(p + "deconv.1.weight"), cp), Epi{}));
    URUN(build_conv(f, id + 4, 3, map_plain(ci), cp, map_plain(cp), ci, W(p + "conv1.0.weight"),
                    vec(W(p + "conv1.0.bias"), cp), vec(W(p + "conv1.1.weight"), cp), Epi{}));
    URUN(build_conv(f, id + 5, 3, map_plain(cp), cp, map_plain(co), cp, W(p + "conv2.0.weight"),
                    vec(W(p + "conv2.0.bias"), co), vec(W(p + "conv2.1.weight"), co), Epi{}));
    if (u == 0) URUN(load_cbam(4, p + "cbam.", co));
  }
  // ---- IFBlocks
  for (int b = 0; b < 3; ++b) {
    const std::string p = "flownet.block" + std::to_string(b) + ".";
    const int C = kBC[b], L = kBL[b], id = kBlk + 8 * b;
    for (int j = 0; j < 6; ++j) {
      const std::string q = p + "convblock." + std::to_string(j) + ".";
      URUN(build_conv(f, id + j, 3, map_plain(C), C, map_plain(C), C, W(q + "0.weight"), vec(W(q + "0.bias"), C),
                      vec(W(q + "1.weight"), C), Epi{}));
    }
    URUN(build_conv(f, id + 6, 3, map_plain(C), C, map_plain(4, 16), C, W(p + "flowconv.weight"),
                    vec(W(p + "flowconv.bias"), 4), none, Epi{2, 0, 4}));
    const std::string mk = p + "maskconvx" + std::to_string(L) + ".";
    URUN(build_conv(f, id + 7, 1, map_plain(C), C, map_plain(9 * L * L, 9 * L * L), C, W(mk + "weight"),
                    vec(W(mk + "bias"), 9 * L * L), none, Epi{0, 0, 0}));
  }
  // ---- RRDBNet
  const std::string fu = "fusionnet.";
  URUN(build_conv(f, kFus, 3, map_plain(16), 64, map_plain(64), 16, W(fu + "conv_first.weight"),
                  vec(W(fu + "conv_first.bias"), 64), none, Epi{0, 0, 0}));
  for (int rr = 0; rr < 6; ++rr)
    for (int d = 0; d < 3; ++d) {
      const std::string q = fu + "body." + std::to_string(rr) + ".rdb" + std::to_string(d + 1) + ".";
      const int id = kFus + 1 + 5 * (3 * rr + d);
      for (int k = 1; k <= 4; ++k) {
        const Map in = map_rdb(k);
        URUN(build_conv(f, id + k - 1, 3, in, 64, map_plain(32, 32), 64 + 32 * (k - 1),
                        W(q + "conv" + std::to_string(k) + ".weight"), vec(W(q + "conv" + std::to_string(k) + ".bias"), 32),
                        none, Epi{0, 1, 0}));
      }
      URUN(build_conv(f, id + 4, 3, map_rdb(5), 64, map_plain(64), 192, W(q + "conv5.weight"),
                      vec(W(q + "conv5.bias"), 64, 0.2f), none, Epi{2, 0, 0}, std::vector<float>(64, 0.2f)));
    }
  URUN(build_conv(f, kFus + 91, 3, map_plain(64), 64, map_plain(64), 64, W(fu + "conv_body.weight"),
                  vec(W(fu + "conv_body.bias"), 64), none, Epi{2, 0, 0}));
  int lid = kFus + 92;
  for (const char* n : {"conv_up1", "conv_up2", "conv_hr"})
    URUN(build_conv(f, lid++, 3, map_plain(64), 64, map_plain(64), 64, W(fu + n + ".weight"), vec(W(fu + n + ".bias"), 64),
                    none, Epi{0, 1, 0}));
  URUN(build_conv(f, kFus + 95, 3, map_plain(64), 64, map_plain(1, 16), 64, W(fu + "conv_last.weight"),
                  vec(W(fu + "conv_last.bias"), 1), none, Epi{2, 0, 2}));
  // ---- ResynNet (conv_bn: BatchNorm folded into the weights and a bias)
  for (int b = 0; b < 3; ++b) {
    const std::string p = "refinenet.block" + std::to_string(b) + ".";
    const int id = kRes + 12 * b, cin0 = b ? 12 : 6;
    auto fold = [&](const std::string& q, int n, std::vector<float>* sc, std::vector<float>* sh) {
      bn_fold(W(q + "1.weight"), W(q + "1.bias"), W(q + "1.running_mean"), W(q + "1.running_var"), n, sc, sh);
    };
    std::vector<float> sc, sh;
    fold(p + "conv0.0.", 64, &sc, &sh);
    std::vector<float> w0(64 * cin0 * 9);
    for (int o = 0; o < 64; ++o)
      for (int j = 0; j < cin0 * 9; ++j) w0[o * cin0 * 9 + j] = W(p + "conv0.0.0.weight")[o * cin0 * 9 + j] * sc[o];
    URUN(upload_f(f, w0, &f->stem[b][0]));
    URUN(upload_f(f, sh, &f->stem[b][1]));
    URUN(upload_f(f, vec(W(p + "conv0.0.2.weight"), 64), &f->stem[b][2]));
    fold(p + "conv0.1.", 128, &sc, &sh);
    URUN(build_conv_s2(f, id, 64, map_plain(128), W(p + "conv0.1.0.weight"), sh, vec(W(p + "conv0.1.2.weight"), 128), sc));
    fold(p + "conv0.2.", 256, &sc, &sh);
    URUN(build_conv_s2(f, id + 1, 128, map_plain(256), W(p + "conv0.2.0.weight"), sh, vec(W(p + "conv0.2.2.weight"), 256),
                       sc));
    for (int j = 0; j < 6; ++j) {
      const std::string q = p + "convblock." + std::to_string(j) + ".";
      fold(q, 256, &sc, &sh);
      URUN(build_conv(f, id + 2 + j, 3, map_plain(256), 256, map_plain(256), 256, W(q + "0.weight"), sh,
                      vec(W(q + "2.weight"), 256), Epi{}, sc));
    }
    URUN(build_convT(f, id + 8, map_plain(256), map_plain(4, 16), 4, W(p + "lastconv.weight"),
                     vec(W(p + "lastconv.bias"), 4), none, Epi{2, 0, 4}));
  }
  for (int k = 0; k < 2; ++k) {
    const std::string p = "refinenet.context" + std::to_string(k) + ".";
    URUN(upload_f(f, vec(W(p + "0.0.weight"), 16 * 27), &f->ctx[k][0]));
    URUN(upload_f(f, vec(W(p + "0.0.bias"), 16), &f->ctx[k][1]));
    URUN(upload_f(f, vec(W(p + "0.1.weight"), 16), &f->ctx[k][2]));
    URUN(build_conv_s2(f, kCtx + k, 16, map_plain(32, 32), W(p + "1.0.weight"), vec(W(p + "1.0.bias"), 32),
                       vec(W(p + "1.1.weight"), 32)));
  }
  URUN(build_convT(f, kDec, map_plain(64), map_plain(32, 64), 32, W("refinenet.decode.0.weight"),
                   vec(W("refinenet.decode.0.bias"), 32), none, Epi{0, 0, 0}));
  URUN(build_convT(f, kDec + 4, map_plain(32), map_plain(3, 16), 3, W("refinenet.decode.1.weight"),
                   vec(W("refinenet.decode.1.bias"), 3), none, Epi{2, 0, 4}));
  f->loaded = true;
  return VFI_OK;
}

int vfi_ifunet_forward(vfi_ctx* c, const float* img0, const float* img1, int H, int W, double timestep, double scale,
                       int ensemble, float* out, void* stream) {
  if (!c || !img0 || !img1 || !out) return ifail(VFI_E_INVALID, "null argument");
  IfunetState* f = state(c);
  if (!f || !f->loaded) return ifail(VFI_E_STATE, "vfi_ifunet_load has not been called");
  if (!std::isfinite(timestep)) return ifail(VFI_E_INVALID, "ifunet: timestep must be finite");
  Geo g{};
  URUN(geometry(H, W, scale, &g));
  UCK(cudaSetDevice(ctx_info(c).device));
  URUN(ensure_workspace(f, g));
  return forward(c, f, img0, img1, g, (float)timestep, ensemble != 0, out, static_cast<cudaStream_t>(stream));
}

int vfi_ifunet_geometry(int H, int W, double scale, int32_t* info, int cap) {
  if (!info) return ifail(VFI_E_INVALID, "ifunet: null argument");
  Geo g{};
  URUN(geometry(H, W, scale, &g));
  int32_t v[14] = {g.Hp, g.Wp};
  for (int l = 0; l < 6; ++l) {
    v[2 + 2 * l] = g.lh[l];
    v[3 + 2 * l] = g.lw[l];
  }
  for (int i = 0; i < cap && i < 14; ++i) info[i] = v[i];
  return VFI_OK;
}

int vfi_ifunet_debug_set_ref(vfi_ctx* c, int use_ref) {
  IfunetState* f = state(c);
  if (!f) return ifail(VFI_E_STATE, "vfi_ifunet_load has not been called");
  f->use_ref = use_ref != 0;
  return VFI_OK;
}

static const StreamConvLayer* ifunet_layer(vfi_ctx* c, int layer) {
  IfunetState* f = state(c);
  if (!f || !f->loaded || layer < 0 || layer >= kNumLayers || !f->conv[layer].w) return nullptr;
  return &f->conv[layer];
}

int vfi_ifunet_debug_conv(vfi_ctx* c, int layer, const void* src0, int pitch0, const void* src1, int pitch1, void* out,
                          int out_pitch, const void* res, float* out_f32, int f32_pitch, int B, int H, int W, int impl,
                          void* stream) {
  const StreamConvLayer* L = ifunet_layer(c, layer);
  if (!L) return ifail(VFI_E_INVALID, "ifunet: no such conv layer (or weights not loaded)");
  UCK(cudaSetDevice(ctx_info(c).device));
  const cudaError_t e = launch_streamconv(*L, state(c)->op_type, src0, pitch0, src1, pitch1, out, out_pitch, B, H, W,
                                          ctx_info(c).num_sms, impl != 0, static_cast<cudaStream_t>(stream), res, out_f32,
                                          f32_pitch);
  ctx_add_launches(c, 1);
  if (e != cudaSuccess) return ifail(VFI_E_CUDA, std::string("streamconv: ") + cudaGetErrorString(e) + " / " + vfi_last_error());
  return VFI_OK;
}

int vfi_ifunet_layer_plan(vfi_ctx* c, int layer, int32_t* info, int cap) {
  const StreamConvLayer* L = ifunet_layer(c, layer);
  if (!L || !info) return ifail(VFI_E_INVALID, "ifunet: no such conv layer (or weights not loaded)");
  StreamConvParams p{};
  if (!streamconv_plan(*L, &p)) return ifail(VFI_E_INVALID, "ifunet: plan failed");
  const int32_t v[14] = {L->c0, L->c1, L->n_total, L->ksize, L->act, L->ext, L->n_f32, -p.halo_y0, -p.halo_x0, p.n_cta,
                         p.nsplit, p.a_slots, p.b_slots, (int32_t)p.smem_bytes};
  for (int i = 0; i < cap && i < 14; ++i) info[i] = v[i];
  return VFI_OK;
}

int vfi_ifunet_debug_elem(vfi_ctx* c, int kernel, const float* img0, const float* img1, int H, int W, double timestep,
                          double scale, const void* x, const void* y, void* out, int index, void* stream) {
  IfunetState* f = state(c);
  if (!f || !f->loaded) return ifail(VFI_E_STATE, "vfi_ifunet_load has not been called");
  if (kernel < 0 || kernel > 3) return ifail(VFI_E_INVALID, "ifunet: no such element-wise kernel");
  UCK(cudaSetDevice(ctx_info(c).device));
  Runner r{f, ctx_info(c), static_cast<cudaStream_t>(stream)};
  const int op = f->op_type;
  switch (kernel) {
    case 0: {  // level-0 input of `index` (1 or 2) images for an H x W frame
      if (index != 1 && index != 2) return ifail(VFI_E_INVALID, "ifunet: flow_in takes 1 or 2 images");
      Geo g{};
      URUN(geometry(H, W, scale, &g));
      const IfuFlowIn a = flow_in_args(f, g, img0, img1, 0, 0, (float)timestep);
      URUN(r.ck(launch_ifunet_flow_in(op, a, index, out, r.st), "flow_in"));
      break;
    }
    case 1: {  // CBAM `index` (0..3: FeatureNet conv2..5, 4: deconv5) in place on out [1][H][W][C]
      if (index < 0 || index > 4) return ifail(VFI_E_INVALID, "ifunet: no such CBAM");
      const int C = index < 4 ? kFC[index + 1] : 256;
      std::vector<float*> tmp(4, nullptr);
      const size_t n[4] = {(size_t)kIfuPoolChunks * C, (size_t)kIfuPoolChunks * C, (size_t)C, (size_t)H * W * 2};
      for (int i = 0; i < 4; ++i) UCK(cudaMalloc(&tmp[i], n[i] * 4));
      const int rc = r.ck(launch_ifunet_cbam(op, out, C, C, 1, H, W, f->cbam_mlp[index], f->cbam_sw[index], tmp[0], tmp[1],
                                             tmp[2], tmp[3], r.st),
                          "cbam");
      cudaStreamSynchronize(r.st);
      for (float* p : tmp) cudaFree(p);
      URUN(rc);
      break;
    }
    case 2: {  // convex upsampling of IFBlock `index`: x = flow fp32 [1][H][W][4], y = mask logits [1][H][W][9 L L]
      if (index < 0 || index > 2) return ifail(VFI_E_INVALID, "ifunet: no such IFBlock");
      URUN(r.ck(launch_ifunet_convex(op, (const float*)x, y, kBL[index], 1, H, W, (float*)out, r.st), "convex"));
      break;
    }
    case 3: {  // warps of an H x W pair by x = flow fp32 [Hp][Wp][4] -> out [2][3][Hp][Wp]
      const int Hp = ((H - 1) / 64 + 1) * 64, Wp = ((W - 1) / 64 + 1) * 64;
      URUN(r.ck(launch_ifunet_warp_frames(img0, img1, H, W, Hp, Wp, (const float*)x, (float*)out, r.st), "warp_frames"));
      break;
    }
  }
  ctx_add_launches(c, r.launches);
  return VFI_OK;
}

}  // extern "C"
