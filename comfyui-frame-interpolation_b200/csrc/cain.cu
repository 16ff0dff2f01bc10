// CAIN (depth 3) on H100: weight packing, the per-geometry workspace, the forward schedule and its C ABI
// (include/vfi_b200.h).  Reference: vfi_models/cain/cain_arch.py, common.py, cain/__init__.py.
//
// Every 3x3 conv of the trunk (Interpolation(5, 12, 192)) is a plain streamconv layer:
//   layer 0                  headConv     cat(x0, x1) as two 192-channel sources, zero padding   ext 0, no activation
//   1 + 25 g + 2 r           RCAB r of group g, conv1                                           ext 0, LeakyReLU(0.2)
//   1 + 25 g + 2 r + 1       RCAB conv2, then channel attention (cain_elem.cu) and + the RCAB input
//   1 + 25 g + 24            group tail conv, + the group input                                 ext 1, slope 1.0
//   126                      tailConv, zero padding                                             ext 0, no activation
//
// Bordered layout.  TMA fills only zeros outside a tensor, and ConvNorm pads by reflection.  So every activation lives on
// an (h + 2) x (w + 2) grid, one cell larger on each side than the h x w trunk grid, and each conv runs over that whole
// grid with streamconv's zero 'same' padding: an interior cell then reads exactly the border the tensor holds.  Before a
// ConvNorm reads a tensor its border holds ReflectionPad2d(1) of the interior; before headConv or tailConv it holds
// zeros.  The border cells a conv writes are invalid until the next border fill or apply overwrites them.  The apply
// kernel writes the whole grid, its border from the mirrored interior cells, so only conv1's output and each group's
// output need a separate border fill.
#include <cuda_fp16.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <cmath>
#include <string>

#include "../../include/vfi_b200.h"
#include "vfi_internal.h"

namespace vfi {

namespace {

constexpr int kC = kCainChannels;
constexpr int kGroups = 5, kBlocks = 12;
constexpr int kNumLayers = 2 + kGroups * (2 * kBlocks + 1);   // 127
constexpr int kTailLayer = kNumLayers - 1;
constexpr int kNumRcab = kGroups * kBlocks;                    // 60
constexpr int kCaFloats = kCainHidden * kC + kCainHidden + kC * kCainHidden + kC;  // W1, b1, W2, b2 of one CALayer

int conv1_id(int g, int r) { return 1 + 25 * g + 2 * r; }
int gtail_id(int g) { return 1 + 25 * g + 2 * kBlocks; }

struct CBuf {
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

struct CainState : ModelState {
  int op_type = OP_F16;
  bool loaded = false;
  bool use_ref = false;  // debug: every conv through the CUDA-core checker
  std::vector<void*> allocs;
  StreamConvLayer conv[kNumLayers];
  float* ca = nullptr;   // [60][kCaFloats]
  // workspace: mean partials, prep output (384 channels), head output, three group / RCAB buffers, conv1 and conv2
  // outputs, attention row sums and gate
  CBuf partial, xin, xh, p[3], t1, t2, sums, gate;
  ~CainState() override {
    for (void* q : allocs) cudaFree(q);
    for (CBuf* b : {&partial, &xin, &xh, &p[0], &p[1], &p[2], &t1, &t2, &sums, &gate}) b->release();
  }
};

namespace {

CainState* state(vfi_ctx* c) { return c ? static_cast<CainState*>(ctx_cain(c)) : nullptr; }

#define CCK(call)                                                            \
  do {                                                                       \
    cudaError_t _e = (call);                                                 \
    if (_e != cudaSuccess) {                                                 \
      set_error(std::string(#call) + ": " + cudaGetErrorString(_e));         \
      return VFI_E_CUDA;                                                     \
    }                                                                        \
  } while (0)

#define CRUN(expr)           \
  do {                       \
    const int _rc = (expr);  \
    if (_rc) return _rc;     \
  } while (0)

int cfail(int code, const std::string& msg) {
  set_error(msg);
  return code;
}

template <class T>
int cupload(CainState* f, const T* h, size_t n, void** dptr) {
  void* d = nullptr;
  CCK(cudaMalloc(&d, n * sizeof(T)));
  f->allocs.push_back(d);
  CCK(cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice));
  *dptr = d;
  return VFI_OK;
}

// Conv2d(cin, 192, 3) weight [192][cin][3][3], cin = 192 or (headConv) 384 read as two 192-channel sources
int build_conv(CainState* f, StreamConvLayer& L, int cin, int act, int ext, const float* w, const float* b) {
  L = StreamConvLayer{};
  L.ksize = 3;
  L.c0 = kC;
  L.c1 = cin - kC;
  L.n_total = kC;
  L.act = act;
  L.ext = ext;
  L.slope = 1.f;
  std::vector<uint16_t> pk;
  StreamConvParams p{};
  if (!pack_streamconv(L, f->op_type, [&](int n, int tap, int j) { return w[((size_t)n * cin + j) * 9 + tap]; }, &pk, &p))
    return cfail(VFI_E_INVALID, "cain: layer shape not supported by streamconv");
  void* d = nullptr;
  CRUN(cupload(f, pk.data(), pk.size(), &d));
  L.w = d;
  CRUN(cupload(f, b, kC, &d));
  L.shift = static_cast<float*>(d);
  return VFI_OK;
}

// ---------------------------------------------------------------- geometry
struct Geo {
  int H, W, Hp, Wp, h, w, top, left;
};

// InOutPaddings: each axis up to a multiple of 128, p // 2 before and p - p // 2 after, by ReflectionPad2d, which needs
// the padding on each side to be smaller than the axis
int geometry(int H, int W, Geo* g) {
  if (H < 1 || W < 1) return cfail(VFI_E_INVALID, "cain: empty frames");
  if (H > 32768 || W > 32768) return cfail(VFI_E_INVALID, "cain: frames larger than 32768 pixels on a side");
  auto pad = [](int n) { return n % 128 == 0 ? 0 : (n / 128 + 1) * 128 - n; };
  const int ph = pad(H), pw = pad(W);
  const int worst_h = ph - ph / 2, worst_w = pw - pw / 2;
  if (worst_h >= H || worst_w >= W)
    return cfail(VFI_E_INVALID, "cain: a " + std::to_string(H) + " x " + std::to_string(W) +
                                    " frame cannot be reflection-padded to a multiple of 128 (padding " +
                                    std::to_string(worst_h >= H ? worst_h : worst_w) + " on one side of a " +
                                    std::to_string(worst_h >= H ? H : W) + "-pixel axis)");
  g->H = H;
  g->W = W;
  g->Hp = H + ph;
  g->Wp = W + pw;
  g->h = g->Hp / 8;
  g->w = g->Wp / 8;
  g->top = ph / 2;
  g->left = pw / 2;
  return VFI_OK;
}

size_t cells(const Geo& g) { return (size_t)(g.h + 2) * (g.w + 2); }

int ensure_workspace(CainState* f, const Geo& g) {
  const size_t t = cells(g) * kC * 2;
  CCK(f->partial.ensure(sizeof(double) * 6 * kCainMeanChunks));
  CCK(f->xin.ensure(2 * t));
  for (CBuf* b : {&f->xh, &f->p[0], &f->p[1], &f->p[2], &f->t1, &f->t2}) CCK(b->ensure(t));
  CCK(f->sums.ensure(sizeof(float) * g.h * kC));
  CCK(f->gate.ensure(sizeof(float) * kC));
  return VFI_OK;
}

struct Runner {
  CainState* f;
  CtxInfo ci;
  cudaStream_t st;
  int launches = 0;
  int ck(cudaError_t e, const char* what) {
    ++launches;
    if (e != cudaSuccess) {
      set_error(std::string("cain: ") + what + ": " + cudaGetErrorString(e) + " / " + vfi_last_error());
      return VFI_E_CUDA;
    }
    return VFI_OK;
  }
  // one conv over the whole bordered grid
  int conv(int id, const void* src, int pitch, void* out, const Geo& g, const void* src1 = nullptr, const void* res = nullptr) {
    return ck(launch_streamconv(f->conv[id], f->op_type, src, pitch, src1, src1 ? pitch : 0, out, kC, 1, g.h + 2, g.w + 2,
                                ci.num_sms, f->use_ref, st, res),
              "streamconv");
  }
  // channel attention of RCAB k on x, + res, into out
  int attention(int k, const void* x, const void* res, void* out, const Geo& g) {
    CRUN(ck(launch_cain_chan_sums(f->op_type, x, g.h, g.w, (float*)f->sums.p, st), "chan_sums"));
    CRUN(ck(launch_cain_gate((const float*)f->sums.p, g.h, g.w, f->ca + (size_t)k * kCaFloats, (float*)f->gate.p, st), "gate"));
    return ck(launch_cain_apply(f->op_type, x, (const float*)f->gate.p, res, out, g.h, g.w, st), "apply");
  }
};

uint8_t* bp(const CBuf& b) { return static_cast<uint8_t*>(b.p); }

int forward(vfi_ctx* c, CainState* f, const float* img0, const float* img1, const Geo& g, float* out, cudaStream_t st) {
  CRUN(ensure_workspace(f, g));
  const int op = f->op_type;
  Runner r{f, ctx_info(c), st};
  double* partial = (double*)f->partial.p;
  // ---- sub_mean, InOutPaddings, pixel_shuffle(1/8), headConv
  CRUN(r.ck(launch_cain_frame_sums(img0, img1, g.H, g.W, partial, st), "frame_sums"));
  CRUN(r.ck(launch_cain_prep(op, img0, img1, g.H, g.W, g.top, g.left, g.h, g.w, partial, f->xin.p, st), "prep"));
  CRUN(r.conv(0, f->xin.p, 2 * kC, f->xh.p, g, bp(f->xin) + kC * 2));
  CRUN(r.ck(launch_cain_border(op, f->xh.p, nullptr, g.h, g.w, true, st), "border"));
  // ---- five residual groups; a group's input stays untouched until its tail conv adds it
  void* gin = f->xh.p;
  for (int gi = 0; gi < kGroups; ++gi) {
    void* cand[2];
    int n = 0;
    for (CBuf& b : f->p)
      if (b.p != gin && n < 2) cand[n++] = b.p;
    void* cur = gin;
    for (int k = 0; k < kBlocks; ++k) {
      const int id = conv1_id(gi, k);
      void* nxt = cur == cand[0] ? cand[1] : cand[0];
      CRUN(r.conv(id, cur, kC, f->t1.p, g));
      CRUN(r.ck(launch_cain_border(op, f->t1.p, nullptr, g.h, g.w, true, st), "border"));
      CRUN(r.conv(id + 1, f->t1.p, kC, f->t2.p, g));
      CRUN(r.attention(gi * kBlocks + k, f->t2.p, cur, nxt, g));
      cur = nxt;
    }
    void* gout = cur == cand[0] ? cand[1] : cand[0];
    CRUN(r.conv(gtail_id(gi), cur, kC, gout, g, nullptr, gin));
    // the next group's ConvNorm needs the reflected border; after the last group, res = body(x) + x with a zero border
    // for tailConv
    const bool last = gi == kGroups - 1;
    CRUN(r.ck(launch_cain_border(op, gout, last ? f->xh.p : nullptr, g.h, g.w, !last, st), "border"));
    gin = gout;
  }
  // ---- tailConv, pixel_shuffle(8), crop, + mean
  CRUN(r.conv(kTailLayer, gin, kC, f->t1.p, g));
  CRUN(r.ck(launch_cain_final(op, f->t1.p, g.H, g.W, g.top, g.left, g.w, partial, out, st), "final"));
  ctx_add_launches(c, r.launches);
  return VFI_OK;
}

// the reference's name of tensor i (state_dict order)
std::string tensor_name(int i) {
  const std::string pre = "encoder.interpolate.";
  if (i < 2) return pre + "headConv." + (i ? "bias" : "weight");
  if (i >= VFI_CAIN_NUM_TENSORS - 2) return pre + "tailConv." + (i % 2 ? "bias" : "weight");
  const int j = i - 2, per_group = kBlocks * 8 + 2, gi = j / per_group, k = j % per_group;
  const std::string gp = pre + "body." + std::to_string(gi) + ".body.";
  if (k >= kBlocks * 8) return gp + std::to_string(kBlocks) + ".conv." + (k % 2 ? "bias" : "weight");
  static const char* kRcab[8] = {"0.conv.weight", "0.conv.bias", "2.conv.weight", "2.conv.bias",
                                 "3.conv_du.0.weight", "3.conv_du.0.bias", "3.conv_du.2.weight", "3.conv_du.2.bias"};
  return gp + std::to_string(k / 8) + ".body." + kRcab[k % 8];
}

int64_t tensor_numel(int i) {
  if (i == 0) return (int64_t)kC * 2 * kC * 9;
  if (i == 1 || i >= VFI_CAIN_NUM_TENSORS - 2) return i % 2 ? kC : (int64_t)kC * kC * 9;
  const int k = (i - 2) % (kBlocks * 8 + 2);
  if (k >= kBlocks * 8) return k % 2 ? kC : (int64_t)kC * kC * 9;
  static const int64_t kRcab[8] = {kC * kC * 9, kC, kC * kC * 9, kC, kCainHidden * kC, kCainHidden, kC * kCainHidden, kC};
  return kRcab[k % 8];
}

}  // namespace
}  // namespace vfi

using namespace vfi;

extern "C" {

/* tensor order: CAIN(depth=3).state_dict() (engine.py cain_state_dict_spec) */
int vfi_cain_load(vfi_ctx* c, const float* const* T, const int64_t* numel, int n_tensors, int operand_type) {
  if (!c || !T || !numel) return cfail(VFI_E_INVALID, "null argument");
  if (n_tensors != VFI_CAIN_NUM_TENSORS)
    return cfail(VFI_E_INVALID, "cain: expected " + std::to_string(VFI_CAIN_NUM_TENSORS) + " tensors, got " +
                                    std::to_string(n_tensors));
  if (operand_type != VFI_OPERAND_F16 && operand_type != VFI_OPERAND_BF16) return cfail(VFI_E_INVALID, "operand type");
  for (int i = 0; i < n_tensors; ++i)
    if (!T[i] || numel[i] != tensor_numel(i))
      return cfail(VFI_E_INVALID, "cain: tensor " + std::to_string(i) + " (" + tensor_name(i) + ") has " +
                                      std::to_string((long long)numel[i]) + " elements, CAIN(depth=3) has " +
                                      std::to_string((long long)tensor_numel(i)));
  const CtxInfo ci = ctx_info(c);
  CCK(cudaSetDevice(ci.device));
  delete ctx_cain(c);
  CainState* f = new CainState();
  ctx_cain(c) = f;
  f->op_type = operand_type;
  CRUN(build_conv(f, f->conv[0], 2 * kC, 0, 0, T[0], T[1]));
  std::vector<float> ca((size_t)kNumRcab * kCaFloats);
  for (int gi = 0; gi < kGroups; ++gi) {
    const int t0 = 2 + gi * (kBlocks * 8 + 2);
    for (int k = 0; k < kBlocks; ++k) {
      const float* const* R = T + t0 + 8 * k;
      CRUN(build_conv(f, f->conv[conv1_id(gi, k)], kC, 1, 0, R[0], R[1]));
      CRUN(build_conv(f, f->conv[conv1_id(gi, k) + 1], kC, 0, 0, R[2], R[3]));
      float* d = ca.data() + (size_t)(gi * kBlocks + k) * kCaFloats;
      for (int j = 4; j < 8; ++j) {
        std::copy(R[j], R[j] + tensor_numel(t0 + 8 * k + j), d);
        d += tensor_numel(t0 + 8 * k + j);
      }
    }
    CRUN(build_conv(f, f->conv[gtail_id(gi)], kC, 0, 1, T[t0 + 8 * kBlocks], T[t0 + 8 * kBlocks + 1]));
  }
  CRUN(build_conv(f, f->conv[kTailLayer], kC, 0, 0, T[n_tensors - 2], T[n_tensors - 1]));
  void* d = nullptr;
  CRUN(cupload(f, ca.data(), ca.size(), &d));
  f->ca = static_cast<float*>(d);
  f->loaded = true;
  return VFI_OK;
}

int vfi_cain_forward(vfi_ctx* c, const float* img0, const float* img1, int H, int W, float* out, void* stream) {
  if (!c || !img0 || !img1 || !out) return cfail(VFI_E_INVALID, "null argument");
  CainState* f = state(c);
  if (!f || !f->loaded) return cfail(VFI_E_STATE, "vfi_cain_load has not been called");
  Geo g{};
  CRUN(geometry(H, W, &g));
  CCK(cudaSetDevice(ctx_info(c).device));
  return forward(c, f, img0, img1, g, out, static_cast<cudaStream_t>(stream));
}

int vfi_cain_geometry(int H, int W, int32_t* info, int cap) {
  if (!info) return cfail(VFI_E_INVALID, "cain: null argument");
  Geo g{};
  CRUN(geometry(H, W, &g));
  const int32_t v[6] = {g.Hp, g.Wp, g.h, g.w, g.top, g.left};
  for (int i = 0; i < cap && i < 6; ++i) info[i] = v[i];
  return VFI_OK;
}

int vfi_cain_debug_set_ref(vfi_ctx* c, int use_ref) {
  CainState* f = state(c);
  if (!f) return cfail(VFI_E_STATE, "vfi_cain_load has not been called");
  f->use_ref = use_ref != 0;
  return VFI_OK;
}

static const StreamConvLayer* cain_layer(vfi_ctx* c, int layer) {
  CainState* f = state(c);
  if (!f || !f->loaded || layer < 0 || layer >= kNumLayers) return nullptr;
  return &f->conv[layer];
}

int vfi_cain_debug_conv(vfi_ctx* c, int layer, const void* src0, int pitch0, const void* src1, int pitch1, void* out,
                        int out_pitch, const void* res, int n_images, int H, int W, int impl, void* stream) {
  const StreamConvLayer* L = cain_layer(c, layer);
  if (!L) return cfail(VFI_E_INVALID, "cain: no such conv layer (or weights not loaded)");
  CCK(cudaSetDevice(ctx_info(c).device));
  const cudaError_t e = launch_streamconv(*L, state(c)->op_type, src0, pitch0, src1, pitch1, out, out_pitch, n_images, H,
                                          W, ctx_info(c).num_sms, impl != 0, static_cast<cudaStream_t>(stream), res);
  ctx_add_launches(c, 1);
  if (e != cudaSuccess) return cfail(VFI_E_CUDA, std::string("streamconv: ") + cudaGetErrorString(e) + " / " + vfi_last_error());
  return VFI_OK;
}

int vfi_cain_layer_plan(vfi_ctx* c, int layer, int32_t* info, int cap) {
  const StreamConvLayer* L = cain_layer(c, layer);
  if (!L || !info) return cfail(VFI_E_INVALID, "cain: no such conv layer (or weights not loaded)");
  StreamConvParams p{};
  if (!streamconv_plan(*L, &p)) return cfail(VFI_E_INVALID, "cain: plan failed");
  const int32_t v[11] = {L->c0, L->c1, L->n_total, L->ksize, L->act, L->ext, p.n_cta, p.nsplit, p.a_slots, p.b_slots,
                         (int32_t)p.smem_bytes};
  for (int i = 0; i < cap && i < 11; ++i) info[i] = v[i];
  return VFI_OK;
}

int vfi_cain_debug_elem(vfi_ctx* c, int kernel, const float* img0, const float* img1, int H, int W, const void* x,
                        const void* res, void* out, int rcab, void* stream) {
  CainState* f = state(c);
  if (!f || !f->loaded) return cfail(VFI_E_STATE, "vfi_cain_load has not been called");
  if (kernel < 0 || kernel > 4) return cfail(VFI_E_INVALID, "cain: no such element-wise kernel");
  if (kernel == 3 && (rcab < 0 || rcab >= kNumRcab)) return cfail(VFI_E_INVALID, "cain: no such RCAB");
  Geo g{};
  CRUN(geometry(H, W, &g));
  CCK(cudaSetDevice(ctx_info(c).device));
  CRUN(ensure_workspace(f, g));
  Runner r{f, ctx_info(c), static_cast<cudaStream_t>(stream)};
  const int op = f->op_type;
  double* partial = (double*)f->partial.p;
  switch (kernel) {
    case 0:
      CRUN(r.ck(launch_cain_frame_sums(img0, img1, H, W, partial, r.st), "frame_sums"));
      CRUN(r.ck(launch_cain_prep(op, img0, img1, H, W, g.top, g.left, g.h, g.w, partial, out, r.st), "prep"));
      break;
    case 1:
      CRUN(r.ck(launch_cain_border(op, out, nullptr, g.h, g.w, true, r.st), "border"));
      break;
    case 2:
      CRUN(r.ck(launch_cain_border(op, out, res, g.h, g.w, false, r.st), "border"));
      break;
    case 3:
      CRUN(r.attention(rcab, x, res, out, g));
      break;
    case 4:
      CRUN(r.ck(launch_cain_frame_sums(img0, img1, H, W, partial, r.st), "frame_sums"));
      CRUN(r.ck(launch_cain_final(op, x, H, W, g.top, g.left, g.w, partial, (float*)out, r.st), "final"));
      break;
  }
  ctx_add_launches(c, r.launches);
  return VFI_OK;
}

}  // extern "C"
