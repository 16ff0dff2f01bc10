// Context, weight repacking, the RIFE-4.6 forward schedule and the C ABI (include/vfi_b200.h).
//
// Forward schedule of one internal pass over B (pair, timestep) tasks - reference IFNet.forward,
// rife_arch.py:465-732, arch "4.6" (blocks (7,192) (12,128) (12,96) (12,64), rife_arch.py:404-408):
//   prep_frames (once per source frame)                       clamp / pad           :476-485
//   for block i, scale s_i:                                                          :519-704
//     front      -> x      [B, Hs/2, Ws/2, 4*16]  16-bit      warp+concat+1/s       :31-70,:238-249,:589-596
//     tapconv    -> c00    [B, Hs/4, Ws/4, 4*c/2] 16-bit      conv0.0 (+lrelu)      :181-184
//     tapconv    -> feat   [B, Hs/4, Ws/4, c]     16-bit      conv0.1 (+lrelu)
//                (4.6's full-resolution block: conv0.0 + conv0.1 as one launch, c00 stays on the SM)
//     8x tapconv -> feat                                       ResConv               :20-28
//     tapconv    -> tmp    [B, Hs, Ws] float4 + float          ConvT+PixelShuffle    :215-218
//     (flow(p) = F(p) + sum_j up(T_j)(p)*s_j: F is stored only by fronts that visit every pixel)  :263-266,:694-696
//   final        -> out [B, H, W, 3] fp32                      warp, sigmoid blend, crop, clamp :703-717,:732
#include <cuda_fp16.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <mutex>
#include <thread>

#include "../../include/vfi_b200.h"
#include "vfi_internal.h"
#include "hoststage.h"

namespace vfi {

static thread_local std::string g_err;
void set_error(const std::string& s) { g_err = s; }

namespace {

const int kBlockC[kMaxBlocks] = {192, 128, 96, 64, 32};  // (the fifth block exists in arch 4.26 only)
const int kBlockCinReal[4] = {7, 12, 12, 12};        // arch 4.6: img0,img1,t | w0,w1,t,mask + flow
const int kBlockCinReal47[4] = {15, 20, 20, 20};     // arch 4.7: + encoded features f0,f1 (4 ch each)
const int kBlockCinReal417[4] = {23, 28, 28, 28};    // arch 4.17: + Head_417 features f0,f1 (8 ch each)
const int kBlockCinReal426[kMaxBlocks] = {15, 28, 28, 28, 28};  // arch 4.26: f0,f1 (4 each) [+ mask, 8 fed-back features, flow]
inline int num_blocks(int arch) { return arch == 426 ? 5 : 4; }

uint16_t to_operand(float v, int op_type) {
  if (op_type == OP_BF16) {
    __nv_bfloat16 h = __float2bfloat16_rn(v);
    uint16_t u;
    std::memcpy(&u, &h, 2);
    return u;
  }
  __half h = __float2half_rn(v);
  uint16_t u;
  std::memcpy(&u, &h, 2);
  return u;
}

// Packed weights = the SWIZZLE_128B K-major wgmma B operand, bit for bit: [split][K16/4 (padded)][n][128-byte row of
// four K=16 steps], 16-byte chunks XOR-swizzled with (n & 7); bulk-copied to shared memory verbatim.
template <class F>
std::vector<uint16_t> pack_weights(const TapConvLayer& L, int op_type, F wfun) {
  const size_t per_split = (size_t)((L.ktotal16 + 3) / 4) * L.n_cta * 64;
  std::vector<uint16_t> v((size_t)L.nsplit * per_split, 0);
  for (int sp = 0; sp < L.nsplit; ++sp) {
    int j = 0;
    for (int e = 0; e < L.ntaps; ++e)
      for (int i = 0; i < L.taps[e].nk16; ++i, ++j)
        for (int c = 0; c < 16; ++c) {
          const int chunk = (j & 3) * 2 + (c >> 3);
          for (int nl = 0; nl < L.n_cta; ++nl) {
            const float val = wfun(e, i * 16 + c, sp * L.n_cta + nl);
            v[sp * per_split + ((size_t)(j >> 2) * L.n_cta + nl) * 64 + (size_t)((chunk ^ (nl & 7)) * 8 + (c & 7))] =
                to_operand(val, op_type);
          }
        }
  }
  return v;
}

// choose the output-channel split: smallest split reaching `want_stages`, else the one with most stages; returns its
// stages (0: no split fits in shared memory)
int choose_split(TapConvLayer& L, const std::vector<int>& splits, int want_stages) {
  int best_split = 1, best_stages = 0;
  for (int sp : splits) {
    if (L.n_total % sp) continue;
    const int nc = L.n_total / sp;
    if (nc % 16) continue;
    L.nsplit = sp;
    L.n_cta = nc;
    TapConvParams p{};
    const int st = tapconv_plan(L, &p);
    if (st >= want_stages) {
      best_split = sp;
      best_stages = st;
      break;
    }
    if (st > best_stages) {
      best_stages = st;
      best_split = sp;
    }
  }
  L.nsplit = best_split;
  L.n_cta = L.n_total / best_split;
  return best_stages;
}

// Tap-conv layer roles.  An IFBlock's layers are vfi_ctx::layers[block][role], numbered as in the C ABI
// (vfi_rife46_debug_layer, vfi_rife46_layer_plan); the Head's layers of arch 4.17 / 4.26 are vfi_ctx::head[].
enum LayerRole : int {
  LAYER_CONV00 = 0,      // conv0.0: stride 2 over the space-to-depth block input, space-to-depth output
  LAYER_CONV01 = 1,      // conv0.1: stride 2 over conv0.0's output
  LAYER_RESCONV = 2,     // the eight ResConvs: LAYER_RESCONV + j, j < 8
  LAYER_LASTCONV = 10,   // ConvTranspose2d + PixelShuffle: flow + mask
  LAYER_LASTFEAT = 11,   // arch 4.26: the 8 feature channels of lastconv, for the next block (not in the last block)
  LAYER_HEAD_CONV = 12,  // Head cnn1 / cnn2: 3x3 + LeakyReLU
  LAYER_HEAD_DECONV,     // Head cnn3: ConvTranspose2d(4, 2, 1), output in space-to-depth form
};
constexpr int kBlockLayers = LAYER_LASTFEAT + 1;

// How a layer of a role with `ch` input channels runs.  A streamed layer (wstream, tapconv.cu) lists its one fixed
// output-channel split; a resident layer takes the first of `splits` whose plan reaches `want_stages` window stages,
// else the one with the most.
struct LayerSpec {
  int epi_mode, out_s2d, wstream;
  std::vector<int> splits;
  int want_stages;
};

LayerSpec layer_spec(int role, int ch) {
  const std::vector<int> div12 = {1, 2, 3, 4, 6, 8, 12};  // the splits of the resident conv0 / ResConv layers
  switch (role) {  // {epi_mode, out_s2d, wstream, splits, want_stages}
    case LAYER_CONV00: return {EPI_BIAS_LRELU, 1, 0, div12, 2};
    case LAYER_CONV01: return {EPI_BIAS_LRELU, 0, 0, div12, 2};
    case LAYER_RESCONV:  // streamed: all channels per CTA up to the wgmma's N = 128, else two halves
      return ch >= 96 ? LayerSpec{EPI_RESCONV, 0, 1, {ch > 128 ? 2 : 1}, 1} : LayerSpec{EPI_RESCONV, 0, 0, div12, 3};
    case LAYER_LASTCONV: return ch == 128 ? LayerSpec{EPI_LASTCONV, 0, 1, {1}, 1} : LayerSpec{EPI_LASTCONV, 0, 0, {1, 5}, 2};
    case LAYER_LASTFEAT: return ch >= 128 ? LayerSpec{EPI_BIAS, 2, 1, {1}, 1} : LayerSpec{EPI_BIAS, 2, 0, {2, 4, 8}, 2};
    case LAYER_HEAD_CONV: return {EPI_BIAS_LRELU, 0, 0, {1}, 2};
    default: return {EPI_BIAS, 0, 0, {1}, 2};  // LAYER_HEAD_DECONV
  }
}

// whether the loaded arch has this block layer: LAYER_LASTFEAT only in arch 4.26, in every block but the last
bool block_has_layer(int arch, int block, int layer) {
  const int nb = num_blocks(arch);
  return block < nb && layer < kBlockLayers && (layer != LAYER_LASTFEAT || (arch == 426 && block + 1 < nb));
}

struct DevBuf {
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
}  // namespace vfi

using namespace vfi;

struct vfi_ctx {
  int device = 0;
  int num_sms = 132;
  int batch = 8;
  int op_type = OP_F16;
  bool loaded = false;
  int64_t launches = 0;
  TapConvLayer layers[kMaxBlocks][kBlockLayers];  // [block][LayerRole]
  std::vector<void*> weight_allocs;
  // workspace
  DevBuf imgs, imgs_h, flow, mask, x, c00, featA, featB, tF[kMaxBlocks], tM[kMaxBlocks], raw, outdev;
  DevBuf tE[kMaxBlocks];         // arch 4.26: block outputs' 8 feature channels [B, Hp/s, Wp/s, 8] 16-bit
  int arch = 46;                 // 46 | 47 (rife47.pth / rife49.pth)
  DevBuf feats, e16;             // arch 4.7: encoded features per source frame (float4), half-res temp
  float* enc[4] = {nullptr, nullptr, nullptr, nullptr};  // encode.0.weight/.bias, encode.1.weight/.bias (fp32)
  TapConvLayer head[3];          // arch 4.17 / 4.26: Head cnn1, cnn2 (+ LeakyReLU), cnn3 (ConvTranspose), 32 (padded) channels
  DevBuf hA, hB;                 // arch 4.17: half-resolution 32-channel scratch of the head (ping-pong)
  int ws_Hp = 0, ws_Wp = 0, ws_B = 0;
  FlowState last_fs{};  // the last pass: its levels, flow / mask planes and which levels those hold (debug_state)
  float4* last_F = nullptr;
  float* last_M = nullptr;
  int last_lo = 0;
  bool last_have_base = false;
  DevBuf dbgF, dbgM;
  cudaStream_t s_h2d = nullptr, s_comp = nullptr, s_d2h = nullptr;
  DevBuf ops_a, ops_b;           // scratch of the channel-last op kernels (splat, 9 x 9 volumes)
  vfi::PinnedBuf pin_in, pin_out;
  // per-kernel-group timing of the forward schedule (vfi_rife_profile): CUDA events recorded on the launching stream
  // around each group while `profile` is set; read (and summed per group id) by vfi_rife_profile_read
  bool profile = false;
  struct ProfSpan { int id; cudaEvent_t e0, e1; };
  std::vector<ProfSpan> prof_spans;  // pinned staging rings of the host-pointer path (pageable caller memory)
  vfi::FilmState* film = nullptr;  // FILM weights and workspace (film.cu)
  vfi::SepState* sep = nullptr;    // Sepconv weights and workspace (sepconv.cu)
  vfi::ModelState* flavr = nullptr;  // FLAVR weights and workspace (flavr.cu)
  vfi::ModelState* ifrnet = nullptr;  // IFRNet weights and workspace (ifrnet.cu)
  vfi::ModelState* cain = nullptr;    // CAIN weights and workspace (cain.cu)
  vfi::ModelState* ifunet = nullptr;  // IFUnet weights and workspace (ifunet.cu)
  bool conv0_unfused = false;  // test hook (vfi_rife46_debug_unfused_conv0): conv0.0 and conv0.1 always as two launches
};

namespace vfi {
CtxInfo ctx_info(::vfi_ctx* c) { return CtxInfo{c->device, c->num_sms, c->s_h2d, c->s_comp, c->s_d2h}; }
FilmState*& ctx_film(::vfi_ctx* c) { return c->film; }
SepState*& ctx_sep(::vfi_ctx* c) { return c->sep; }
ModelState*& ctx_flavr(::vfi_ctx* c) { return c->flavr; }
ModelState*& ctx_ifrnet(::vfi_ctx* c) { return c->ifrnet; }
ModelState*& ctx_cain(::vfi_ctx* c) { return c->cain; }
ModelState*& ctx_ifunet(::vfi_ctx* c) { return c->ifunet; }
void ctx_add_launches(::vfi_ctx* c, int n) { c->launches += n; }
}  // namespace vfi

namespace {

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t _e = (call);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      set_error(std::string(#call) + ": " + cudaGetErrorString(_e));                               \
      return VFI_E_CUDA;                                                                           \
    }                                                                                              \
  } while (0)

int fail(int code, const std::string& msg) {
  set_error(msg);
  return code;
}

void free_weights(vfi_ctx* c) {
  for (void* p : c->weight_allocs) cudaFree(p);
  c->weight_allocs.clear();
  c->loaded = false;
}

template <class T>
int upload(vfi_ctx* c, const std::vector<T>& h, void** dptr) {
  void* d = nullptr;
  CK(cudaMalloc(&d, h.size() * sizeof(T)));
  c->weight_allocs.push_back(d);
  CK(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
  *dptr = d;
  return VFI_OK;
}

// A layer's weights as a function of (kernel tap ky*3 + kx, input channel, output column), and its shift per column.
struct WeightMap {
  std::function<float(int tap, int ci, int n)> w;
  std::function<float(int n)> shift;
};

// Conv2d(creal -> nreal, 3x3) [nreal][creal][3][3] + bias; input channels and columns past the real ones are zero
// padding.  `beta` (ResConv): (conv(x) + b) * beta + x == conv_{w*beta}(x) + b*beta + x - beta is folded into the packed
// weights (one 16-bit rounding of w*beta instead of w) so the epilogue is a pure add.
WeightMap conv2d(const float* w, const float* bias, int creal, int nreal, const float* beta = nullptr) {
  return {[=](int tap, int ci, int n) {
            return ci < creal && n < nreal ? w[((size_t)n * creal + ci) * 9 + tap] * (beta ? beta[n] : 1.f) : 0.f;
          },
          [=](int n) { return n < nreal ? bias[n] * (beta ? beta[n] : 1.f) : 0.f; }};
}

// Column n of a ConvTranspose2d(4, 2, 1) run as a 3x3 tap conv: channel oc at sub-pixel (a, b) of the 2x2 block an input
// cell (y, x) covers, output position (2y + a, 2x + b).
struct ConvTCol { int oc, a, b; };

// ConvTranspose2d(creal -> cout, 4, 2, 1) [creal][cout][4][4] + bias as ONE 3x3 conv on the input grid: tap (dy, dx)
// of column n uses transposed-kernel element ky = a+1-2dy, kx = b+1-2dx (no weight outside the 4x4 kernel).
WeightMap conv_transpose(const float* wt, const float* bias, int creal, int cout, std::function<ConvTCol(int)> col) {
  return {[=](int tap, int ci, int n) {
            const ConvTCol k = col(n);
            const int ky = k.a + 1 - 2 * (tap / 3 - 1), kx = k.b + 1 - 2 * (tap % 3 - 1);
            if (ci >= creal || ky < 0 || ky > 3 || kx < 0 || kx > 3) return 0.f;
            return wt[(((size_t)ci * cout + k.oc) * 4 + ky) * 4 + kx];
          },
          [=](int n) { return bias[col(n).oc]; }};
}

// ConvTranspose2d + PixelShuffle(2): channel c at sub-pixel (py, px) of an input cell's 4x4 patch
ConvTCol shuffled(int c, int py, int px) { return {4 * c + 2 * (py & 1) + (px & 1), py >> 1, px >> 1}; }

// One tap-conv layer of `role` over `ch` input channels (conv0.0 / conv0.1: per space-to-depth sub-pixel) with n_total
// output columns: its taps, the plan of layer_spec, and its packed weights and shift uploaded.
int build_layer(vfi_ctx* c, TapConvLayer& L, int role, int ch, int n_total, const WeightMap& wm) {
  const LayerSpec s = layer_spec(role, ch);
  const bool s2 = role == LAYER_CONV00 || role == LAYER_CONV01;
  // a streamed layer over whole 64-channel k-blocks takes k-block-major (kb, tap) entries, else one entry per tap over all
  // channels; the packed weights follow the same K order
  const int nkb = s.wstream && ch % 64 == 0 ? ch / 64 : 1;
  L = TapConvLayer{};
  L.cin = s2 ? 4 * ch : ch;
  L.n_total = n_total;
  L.ntaps = 9 * nkb;
  L.ktotal16 = 9 * (ch / 16);
  L.halo_y0 = -1; L.halo_x0 = -1; L.halo_h = kTileH + (s2 ? 1 : 2); L.halo_w = kTileW + (s2 ? 1 : 2);
  L.epi_mode = s.epi_mode;
  L.out_s2d = s.out_s2d;
  L.wstream = s.wstream;
  for (int kb = 0; kb < nkb; ++kb)
    for (int e = 0; e < 9; ++e) {
      TapEntry& t = L.taps[kb * 9 + e];
      const int ky = e / 3, kx = e % 3;
      t.nk16 = (int16_t)(ch / 16 / nkb);
      if (s2) {  // input row 2y + ky - 1 = 2(y + dy) + a: space-to-depth row offset dy, sub-row a (columns alike)
        const int a = ky == 0 ? 1 : ky - 1, b = kx == 0 ? 1 : kx - 1;
        t.dy = (int16_t)(ky == 0 ? -1 : 0); t.dx = (int16_t)(kx == 0 ? -1 : 0);
        t.chunk0 = (int16_t)((a * 2 + b) * ch / 8);
      } else {
        t.dy = (int16_t)(ky - 1); t.dx = (int16_t)(kx - 1);
        t.chunk0 = (int16_t)(kb * 8);
      }
    }
  const int real_taps = L.ntaps;
  if (s.wstream && (L.ktotal16 & 3)) {  // zero-weight K=16 steps complete the last four-step weight slot (c = 96: 54 + 2)
    TapEntry& t = L.taps[L.ntaps++];  // dy = dx = chunk0 = 0
    t.nk16 = (int16_t)(4 - (L.ktotal16 & 3));
    L.ktotal16 += t.nk16;
  }
  if (choose_split(L, s.splits, s.want_stages) < 1) return fail(VFI_E_STATE, "a layer has no shared-memory plan");
  std::vector<uint16_t> pk = pack_weights(L, c->op_type, [&](int e, int ci, int n) {  // ci relative to the k-block
    return e < real_taps ? wm.w(e % 9, (e / 9) * 64 + ci, n) : 0.f;
  });
  std::vector<float> sh(n_total);
  for (int n = 0; n < n_total; ++n) sh[n] = wm.shift(n);
  int r;
  if ((r = upload(c, pk, &L.w))) return r;
  return upload(c, sh, (void**)&L.shift);
}

struct Geometry {
  int Hp, Wp;
  int nb;  // blocks: 4, arch 4.26: 5
  int s[kMaxBlocks];  // block scale (>= 1); 1 for an up-scaled block
  int k[kMaxBlocks];  // 1, or the up-scaling factor 2 / 4 of a block whose scale is 1/k (node scale_factor 2 / 4)
  // first block whose front visits every full-resolution pixel (scale <= 2, or up-scaled); the blocks before it are the
  // "coarse" blocks, which run over a whole coarse span of pairs (forward_span)
  int dense;
  size_t level_px(int i) const { return (size_t)(Hp * k[i] / s[i]) * (Wp * k[i] / s[i]); }  // block i's grid, per pair
};

int make_geometry(int arch, int H, int W, float scale_factor, Geometry* g) {
  g->Hp = ((H - 1) / 64 + 1) * 64;  // rife_arch.py:480-482
  g->Wp = ((W - 1) / 64 + 1) * 64;
  g->nb = num_blocks(arch);
  for (int i = 0; i < g->nb; ++i) {
    const float sf = (float)(1 << (g->nb - 1 - i)) / scale_factor;  // [8,4,2,1] or [16,8,4,2,1] / scale_factor, rife/__init__.py:156-160
    g->k[i] = 1;
    if (sf < 1.f) {  // a block that UP-scales its input by k = 1 / scale (scale_factor 2: last block, 4: last two)
      const int ki = (int)std::lround(1.f / sf);
      if (std::fabs(1.f / sf - (float)ki) > 1e-6f || (ki != 2 && ki != 4))
        return fail(VFI_E_INVALID, "scale_factor must be one of 0.25, 0.5, 1, 2, 4");
      g->k[i] = ki;
      g->s[i] = 1;
      continue;
    }
    const int si = (int)std::lround(sf);
    if (std::fabs(sf - (float)si) > 1e-6f || si < 1 || (si & (si - 1)))
      return fail(VFI_E_INVALID, "scale_factor must be one of 0.25, 0.5, 1, 2, 4");
    g->s[i] = si;
    if ((g->Hp / si) % 4 || (g->Wp / si) % 4 || g->Hp % si || g->Wp % si)
      return fail(VFI_E_INVALID,
                  "padded size / scale is not a multiple of 4: the reference fails with a shape mismatch for this "
                  "size and scale_factor as well");
  }
  g->dense = g->nb;
  for (int i = g->nb - 1; i >= 1; --i)
    if (g->s[i] <= 2) g->dense = i;
  return VFI_OK;
}

// Workspace bytes of block i per pair: its s2d block input (x), conv0.0 output (c00), one ResConv feature map (featA / featB
// each) and its output level (tF, tM and arch 4.26's tE).
struct BlockBytes { size_t x, c00, feat, level; };

BlockBytes block_bytes(const vfi_ctx* c, const Geometry& g, int i) {
  const size_t px = g.level_px(i);
  return {px / 4 * (c->arch != 46 ? 128 : 64) * 2, px / 16 * 2 * kBlockC[i] * 2, px / 16 * kBlockC[i] * 2,
          px * (sizeof(float4) + sizeof(float) + (block_has_layer(c->arch, i, LAYER_LASTFEAT) ? 16 : 0))};
}

// Byte budgets of the wide spans (workspace at the blocks' own sizes: the shared x / c00 / featA / featB plus the output
// levels, and for the first dense block the full-resolution flow / mask planes it stores).  At 1080p the coarse blocks of
// 4.6 cost 15.8 MB per pair, so 1 GiB holds one span of a whole 63-pair forward call; the first dense block (block 2 of
// 4.6, scale 2) costs 169 MB per pair, so 4 GiB holds spans of 24 pairs (DESIGN.md section 4.3 has the measured widths).
// A build may set other budgets (the host-emulation tests use a few hundred kB, so that tiny frames take several spans).
#ifndef VFI_COARSE_BUDGET_BYTES
#define VFI_COARSE_BUDGET_BYTES (1ull << 30)
#endif
#ifndef VFI_MID_BUDGET_BYTES
#define VFI_MID_BUDGET_BYTES (4ull << 30)
#endif
constexpr size_t kCoarseBudget = VFI_COARSE_BUDGET_BYTES;
constexpr size_t kMidBudget = VFI_MID_BUDGET_BYTES;

// How many pairs each block runs over per launch.  The coarse blocks [0, g.dense) run over coarse spans of Bc pairs; the
// first dense block, when another block follows it, over middle spans of Bm pairs inside them; the other blocks and
// `final` over passes of B = `batch` pairs inside those (a middle span ends early where its coarse span ends).  Bc and Bm
// are whole numbers of B, so the passes fall where they would if every block ran pass by pass.
struct Widths {
  int Bc, Bm, B;
  int dense;  // g.dense
  int mid;    // g.dense when that block runs over middle spans, else -1 (it is the last block, or up-scaled; Bm = B)
  int of(int i) const { return i < dense ? Bc : i == mid ? Bm : B; }
};

// The most pairs whose bytes per pair fit `budget`, as a whole number of `unit`, at least `unit` and at most n_tasks
int fit_width(size_t per_pair, size_t budget, int unit, int n_tasks) {
  const int fit = (int)std::min<size_t>(budget / per_pair, 1 << 20);
  return std::min(n_tasks, std::max(unit, fit / unit * unit));
}

Widths span_widths(const vfi_ctx* c, const Geometry& g, int B, int n_tasks) {
  Widths w{B, B, B, g.dense, -1};
  if (g.dense + 1 < g.nb && g.k[g.dense] == 1) {
    const BlockBytes b = block_bytes(c, g, g.dense);
    const size_t per_pair = b.x + b.c00 + 2 * b.feat + b.level + (size_t)g.Hp * g.Wp * (sizeof(float4) + sizeof(float));
    w.mid = g.dense;
    w.Bm = fit_width(per_pair, kMidBudget, B, n_tasks);
  }
  size_t x = 0, c00 = 0, feat = 0, level = 0;
  for (int i = 0; i < g.dense; ++i) {
    const BlockBytes b = block_bytes(c, g, i);
    x = std::max(x, b.x);
    c00 = std::max(c00, b.c00);
    feat = std::max(feat, b.feat);
    level += b.level;
  }
  w.Bc = fit_width(x + c00 + 2 * feat + level, kCoarseBudget, B, n_tasks);
  return w;
}

int ensure_workspace(vfi_ctx* c, const Geometry& g, const Widths& w, int n_frames_window) {
  size_t x = 0, c00 = 0, feat = 0;
  for (int i = 0; i < g.nb; ++i) {
    const size_t n = w.of(i);
    const BlockBytes b = block_bytes(c, g, i);
    const size_t px = n * g.level_px(i);
    x = std::max(x, n * b.x);
    c00 = std::max(c00, n * b.c00);
    feat = std::max(feat, n * b.feat);
    CK(c->tF[i].ensure(px * sizeof(float4)));  // block output T_i (flow increments at 1/s_i)
    CK(c->tM[i].ensure(px * sizeof(float)));
    if (block_has_layer(c->arch, i, LAYER_LASTFEAT)) CK(c->tE[i].ensure(px * 16));
  }
  const size_t px = (size_t)g.Hp * g.Wp;
  CK(c->imgs.ensure((size_t)n_frames_window * px * sizeof(float4)));
  CK(c->imgs_h.ensure((size_t)n_frames_window * px * sizeof(uint2)));
  if (c->arch == 47) {
    CK(c->feats.ensure((size_t)n_frames_window * px * sizeof(uint2)));  // half4 features
    CK(c->e16.ensure((size_t)(kMaxBatch + 2) * (px / 4) * 16 * sizeof(float)));
  }
  if (c->arch == 417 || c->arch == 426) {
    // features: 8 (4.26: 4) x 16-bit per pixel, space-to-depth cells of 32 (16) values; head scratch: 32 ch at 1/2 res
    CK(c->feats.ensure((size_t)n_frames_window * px * (c->arch == 417 ? 16 : 8)));
    CK(c->hA.ensure((size_t)(kMaxBatch + 2) * (px / 4) * 32 * 2));
    CK(c->hB.ensure((size_t)(kMaxBatch + 2) * (px / 4) * 32 * 2));
  }
  CK(c->flow.ensure((size_t)std::max(w.Bm, w.B) * px * sizeof(float4)));  // written by the first dense block onwards
  CK(c->mask.ensure((size_t)std::max(w.Bm, w.B) * px * sizeof(float)));
  CK(c->x.ensure(x));
  CK(c->c00.ensure(c00));
  CK(c->featA.ensure(feat));
  CK(c->featB.ensure(feat));
  c->ws_Hp = g.Hp;
  c->ws_Wp = g.Wp;
  return VFI_OK;
}

#define LAUNCH(call)                                               \
  do {                                                             \
    cudaError_t _e = (call);                                       \
    c->launches++;                                                 \
    if (_e != cudaSuccess) {                                       \
      set_error(std::string(#call) + ": " + cudaGetErrorString(_e)); \
      return VFI_E_CUDA;                                           \
    }                                                              \
  } while (0)

// encode head of arch 4.7 / 4.17 for frames [f, f + n) of the prepared window (n <= kMaxBatch + 2), once per source frame
int run_encode(vfi_ctx* c, const Geometry& g, int f, int n, cudaStream_t st) {
  const size_t px = (size_t)g.Hp * g.Wp;
  const float4* imgs = (const float4*)c->imgs.p + (size_t)f * px;
  if (c->arch == 47) {
    LAUNCH(launch_encode(imgs, c->enc[0], c->enc[1], c->enc[2], c->enc[3], (float*)c->e16.p,
                         (uint2*)c->feats.p + (size_t)f * px, n, g.Hp, g.Wp, st));
  } else if (c->arch == 417 || c->arch == 426) {
    const int Hh = g.Hp / 2, Wh = g.Wp / 2;
    const size_t fbytes = c->arch == 417 ? 16 : 8;  // feature bytes per full-resolution pixel
    LAUNCH(launch_head0(c->op_type, imgs, c->enc[0], c->enc[1], c->hA.p, n, g.Hp, g.Wp, st));
    LAUNCH(launch_tapconv(c->head[0], c->op_type, c->hA.p, c->hB.p, nullptr, nullptr, n, Hh, Wh, c->num_sms,
                          TAPCONV_PLANNED, st));
    LAUNCH(launch_tapconv(c->head[1], c->op_type, c->hB.p, c->hA.p, nullptr, nullptr, n, Hh, Wh, c->num_sms,
                          TAPCONV_PLANNED, st));
    LAUNCH(launch_tapconv(c->head[2], c->op_type, c->hA.p, (uint8_t*)c->feats.p + (size_t)f * px * fbytes, nullptr, nullptr,
                          n, Hh, Wh, c->num_sms, TAPCONV_PLANNED, st));
  }
  return VFI_OK;
}

// Whether block i runs conv0.0 and conv0.1 as one launch (launch_conv0_fused): arch 4.6's 64-channel block at full
// resolution, the block whose conv0.0 output is too large to stay in L2 between two launches.  Elsewhere that output is
// small and largely L2-resident, and the 128-channel block inputs of the other archs do not fit the fused kernel's window.
bool conv0_fused(const vfi_ctx* c, const Geometry& g, int i) {
  return !c->conv0_unfused && c->arch == 46 && g.s[i] == 1 && g.k[i] == 1 &&
         conv0_fused_plan(c->layers[i][LAYER_CONV00], c->layers[i][LAYER_CONV01], c->op_type, nullptr, nullptr, nullptr) > 0;
}

// group ids of vfi_rife_profile: 10 * block + {0 front, 1 conv0.0, 2 conv0.1, 3 the 8 ResConvs, 4 lastconv(s)}, 90 final.
// A block that runs conv0.0 and conv0.1 as one launch records it as group 10 * block + 1 and has no group 10 * block + 2.
// A coarse block's spans cover its whole coarse span of pairs, a dense block's one pass.
void span_begin(vfi_ctx* c, int id, cudaStream_t st) {
  if (!c->profile) return;
  vfi_ctx::ProfSpan sp{id, nullptr, nullptr};
  cudaEventCreate(&sp.e0);
  cudaEventCreate(&sp.e1);
  cudaEventRecord(sp.e0, st);
  c->prof_spans.push_back(sp);
}

void span_end(vfi_ctx* c, cudaStream_t st) {
  if (c->profile) cudaEventRecord(c->prof_spans.back().e1, st);
}

// The tasks of a forward span: frame indices into the prepared frame window c->imgs, and timesteps
struct SpanTasks {
  const int32_t* f0;
  const int32_t* f1;
  const float* t;
  BatchTasks batch(int pos, int n) const {  // n <= kMaxBatch
    BatchTasks bt{};
    bt.n = n;
    for (int i = 0; i < n; ++i) {
      bt.f0[i] = f0[pos + i];
      bt.f1[i] = f1[pos + i];
      bt.t[i] = t[pos + i];
    }
    return bt;
  }
};

// The block output levels (4.26: and feature levels) and the full-resolution flow / mask planes, seen from one pair
struct Levels {
  FlowState fs;
  uint8_t* e[kMaxBlocks];  // arch 4.26: tE
  float4* F;               // accumulated full-resolution flow / mask, written only by "dense" fronts
  float* M;
};

// lv with levels [0, upto) advanced by p pairs, and with `planes` the flow / mask planes too
Levels advance(Levels lv, const Geometry& g, int upto, bool planes, int p) {
  for (int j = 0; j < upto; ++j) {
    lv.fs.f[j] += (size_t)p * g.level_px(j);
    lv.fs.m[j] += (size_t)p * g.level_px(j);
    if (lv.e[j]) lv.e[j] += (size_t)p * g.level_px(j) * 16;
  }
  if (planes) {
    lv.F += (size_t)p * g.Hp * g.Wp;
    lv.M += (size_t)p * g.Hp * g.Wp;
  }
  return lv;
}

// Block i over the n pairs tk[pos, pos + n): its front, then conv0.0, conv0.1, the 8 ResConvs and lastconv (4.26: and the
// feature conv), each one tap-conv launch over all n pairs.  lv: the earlier levels and the flow / mask planes at pair `pos`;
// block i's own level is written from its first pair.  lo / have_base: which levels the flow / mask planes hold, read and
// advanced by dense and up-scaled fronts.  A front runs in chunks of at most kMaxBatch tasks (BatchTasks); a chunk at pair
// `at` writes the block input and reads and writes the earlier levels and the planes there.
int run_block(vfi_ctx* c, const Geometry& g, int i, const SpanTasks& tk, int pos, int n, const Levels& lv, int& lo,
              bool& have_base, cudaStream_t st) {
  const float4* imgs = (const float4*)c->imgs.p;
  const uint2* imgs_h = (const uint2*)c->imgs_h.p;
  const void* feats = c->arch != 46 ? c->feats.p : nullptr;
  const FlowState& fs = lv.fs;
  const int s = g.s[i];
  const int Hs = g.Hp * g.k[i] / s, Ws = g.Wp * g.k[i] / s;
  const int ps = i > 0 ? g.s[i - 1] : 1;
  const bool dense = i >= g.dense;
  span_begin(c, 10 * i, st);
  if (g.k[i] > 1) {
    // up-scaled block: fold every level so far into the dense planes, build the k-times finer input from them
    if (i == 0) return fail(VFI_E_INVALID, "the first block cannot be up-scaled");
    if (n > kMaxBatch) return fail(VFI_E_STATE, "an up-scaled block runs at most 16 pairs at once");
    if (lo < i) {
      FlowState part = fs;
      part.n = i;
      LAUNCH(launch_materialize(part, lo, have_base ? lv.F : nullptr, have_base ? lv.M : nullptr, lv.F, lv.M, n, g.Hp, g.Wp,
                                st));
      have_base = true;
      lo = i;
    }
    LAUNCH(launch_front_up(c->op_type, c->arch, imgs_h, feats, i > 0 ? lv.e[i - 1] : nullptr, ps, g.k[i - 1], lv.F, lv.M,
                           tk.batch(pos, n), g.Hp, g.Wp, g.k[i], c->x.p, st));
  } else {
    // a dense front stores the accumulated flow, the last one too: `final` adding two levels per pixel is instruction bound
    const size_t x_pair = block_bytes(c, g, i).x;
    for (int at = 0; at < n; at += kMaxBatch) {
      const Levels ck = advance(lv, g, i, true, at);
      LAUNCH(launch_front(c->op_type, c->arch, imgs, imgs_h, feats, i > 0 ? ck.e[i - 1] : nullptr, ps, ck.fs, i,
                          dense ? lo : 0, dense && have_base ? ck.F : nullptr, dense && have_base ? ck.M : nullptr,
                          dense ? ck.F : nullptr, dense ? ck.M : nullptr, tk.batch(pos + at, std::min(kMaxBatch, n - at)),
                          g.Hp, g.Wp, s, (uint8_t*)c->x.p + at * x_pair, st));
    }
    if (dense) {
      have_base = true;
      lo = i;
    }
  }
  span_end(c, st);
  span_begin(c, 10 * i + 1, st);
  if (conv0_fused(c, g, i)) {
    LAUNCH(launch_conv0_fused(c->layers[i][LAYER_CONV00], c->layers[i][LAYER_CONV01], c->op_type, c->x.p, c->c00.p,
                              c->featA.p, n, Hs / 2, Ws / 2, c->num_sms, st));
    span_end(c, st);
  } else {
    LAUNCH(launch_tapconv(c->layers[i][LAYER_CONV00], c->op_type, c->x.p, c->c00.p, nullptr, nullptr, n, Hs / 2, Ws / 2,
                          c->num_sms, TAPCONV_PLANNED, st));
    span_end(c, st);
    span_begin(c, 10 * i + 2, st);
    LAUNCH(launch_tapconv(c->layers[i][LAYER_CONV01], c->op_type, c->c00.p, c->featA.p, nullptr, nullptr, n, Hs / 4,
                          Ws / 4, c->num_sms, TAPCONV_PLANNED, st));
    span_end(c, st);
  }
  void* a = c->featA.p;
  void* b = c->featB.p;
  span_begin(c, 10 * i + 3, st);
  for (int j = 0; j < 8; ++j) {
    LAUNCH(launch_tapconv(c->layers[i][LAYER_RESCONV + j], c->op_type, a, b, nullptr, nullptr, n, Hs / 4, Ws / 4, c->num_sms,
                          TAPCONV_PLANNED, st));
    std::swap(a, b);
  }
  span_end(c, st);
  span_begin(c, 10 * i + 4, st);
  LAUNCH(launch_tapconv(c->layers[i][LAYER_LASTCONV], c->op_type, a, nullptr, fs.f[i], fs.m[i], n, Hs / 4, Ws / 4, c->num_sms,
                        TAPCONV_PLANNED, st));
  if (block_has_layer(c->arch, i, LAYER_LASTFEAT))  // the 8 feature channels of lastconv, for the next block's input
    LAUNCH(launch_tapconv(c->layers[i][LAYER_LASTFEAT], c->op_type, a, lv.e[i], nullptr, nullptr, n, Hs / 4, Ws / 4,
                          c->num_sms, TAPCONV_PLANNED, st));
  if (g.k[i] > 1) {  // the up-scaled block's output goes straight back onto the dense planes
    LAUNCH(launch_fold_down(fs.f[i], fs.m[i], g.k[i], lv.F, lv.M, n, g.Hp, g.Wp, fs.mask_replace, st));
    lo = i + 1;
  }
  span_end(c, st);
  return VFI_OK;
}

// One coarse span: tasks tk[0, n) -> out [n, H, W, 3], n <= w.Bc.  The coarse blocks (before g.dense) run over all n pairs
// at once, so that their small grids fill the GPU; the first dense block over middle spans of w.Bm pairs; the other blocks
// and `final` in passes of w.B pairs.  Per-pair arithmetic does not depend on how many pairs a launch covers, so the frames
// are the same for any widths.  The workspace holds each block's width of pairs (ensure_workspace).
int forward_span(vfi_ctx* c, const Geometry& g, const SpanTasks& tk, int n, const Widths& w, int H, int W, float* out,
                 cudaStream_t st) {
  Levels lv{};
  lv.fs.n = g.nb;
  for (int i = 0; i < g.nb; ++i) {
    lv.fs.f[i] = (float4*)c->tF[i].p;
    lv.fs.m[i] = (float*)c->tM[i].p;
    lv.fs.s[i] = g.s[i];
    lv.e[i] = (uint8_t*)c->tE[i].p;
  }
  lv.fs.mask_replace = (c->arch != 46) ? 1 : 0;
  lv.F = (float4*)c->flow.p;
  lv.M = (float*)c->mask.p;
  int r, lo = 0;  // levels [lo, i) are not yet folded into the dense planes
  bool have_base = false;
  for (int i = 0; i < g.dense; ++i)
    if ((r = run_block(c, g, i, tk, 0, n, lv, lo, have_base, st))) return r;
  const int mid_end = w.mid >= 0 ? w.mid + 1 : g.dense;
  for (int mpos = 0; mpos < n; mpos += w.Bm) {
    const int mn = std::min(w.Bm, n - mpos);
    const Levels ml = advance(lv, g, g.dense, false, mpos);  // the coarse levels from this middle span's first pair
    int mlo = lo;
    bool mbase = have_base;
    for (int i = g.dense; i < mid_end; ++i)
      if ((r = run_block(c, g, i, tk, mpos, mn, ml, mlo, mbase, st))) return r;
    for (int pos = 0; pos < mn; pos += w.B) {
      const int nb = std::min(w.B, mn - pos);
      const Levels pl = advance(ml, g, mid_end, true, pos);  // every wider level and the planes from this pass's first pair
      int plo = mlo;
      bool pbase = mbase;
      for (int i = mid_end; i < g.nb; ++i)
        if ((r = run_block(c, g, i, tk, mpos + pos, nb, pl, plo, pbase, st))) return r;
      span_begin(c, 90, st);
      LAUNCH(launch_final((const float4*)c->imgs.p, pl.fs, plo, pbase ? pl.F : nullptr, pbase ? pl.M : nullptr,
                          tk.batch(mpos + pos, nb), g.Hp, g.Wp, H, W, out + (size_t)(mpos + pos) * H * W * 3, st));
      span_end(c, st);
      c->last_fs = pl.fs;
      c->last_F = pl.F;
      c->last_M = pl.M;
      c->last_lo = plo;
      c->last_have_base = pbase;
      c->ws_B = nb;
    }
  }
  return VFI_OK;
}

int check_tasks(const int32_t* f0, const int32_t* f1, int n_tasks, int lo, int hi) {
  for (int i = 0; i < n_tasks; ++i)
    if (f0[i] < lo || f0[i] >= hi || f1[i] < lo || f1[i] >= hi) return fail(VFI_E_INVALID, "task frame index out of range");
  return VFI_OK;
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

const char* vfi_last_error(void) { return g_err.c_str(); }
const char* vfi_version(void) { return "vfi_b200 0.3 (sm_90a; RIFE 4.6/4.7/4.17/4.26, FILM, Sepconv, GMFSS Fortuna building blocks; built " __DATE__ " " __TIME__ ")"; }

int vfi_create(int device, vfi_ctx** out) {
  if (!out) return fail(VFI_E_INVALID, "null out");
  int n = 0;
  CK(cudaGetDeviceCount(&n));
  if (device < 0 || device >= n) return fail(VFI_E_INVALID, "no such CUDA device");
  CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9) return fail(VFI_E_INVALID, "libvfi_b200 needs a compute-capability 9.x (H100, sm_90a) GPU");
  vfi_ctx* c = new vfi_ctx();
  c->device = device;
  c->num_sms = prop.multiProcessorCount;
  {
    // VFI_NUM_SMS=n: size the persistent grids for n SMs (an even number, at least 2), leaving the rest to kernels of other
    // streams - e.g. NCCL's receive kernels on the rank that gathers every other rank's frames
    const int want = env_int("VFI_NUM_SMS", 0, 0, 4096);
    if (want >= 2 && want < c->num_sms) c->num_sms = want & ~1;
  }
  CK(cudaStreamCreateWithFlags(&c->s_h2d, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&c->s_comp, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&c->s_d2h, cudaStreamNonBlocking));
  *out = c;
  return VFI_OK;
}

int vfi_destroy(vfi_ctx* c) {
  if (!c) return VFI_OK;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  free_weights(c);
  film_destroy(c->film);
  delete c->flavr;
  c->flavr = nullptr;
  delete c->ifrnet;
  c->ifrnet = nullptr;
  delete c->cain;
  c->cain = nullptr;
  delete c->ifunet;
  c->ifunet = nullptr;
  c->film = nullptr;
  sepconv_destroy(c->sep);
  c->sep = nullptr;
  for (DevBuf* b : {&c->imgs, &c->imgs_h, &c->flow, &c->mask, &c->x, &c->c00, &c->featA, &c->featB, &c->raw, &c->outdev, &c->feats, &c->e16, &c->hA, &c->hB, &c->dbgF,
                    &c->dbgM, &c->ops_a, &c->ops_b})
    b->release();
  for (int i = 0; i < kMaxBlocks; ++i) {
    c->tF[i].release();
    c->tM[i].release();
    c->tE[i].release();
  }
  c->pin_in.release();
  c->pin_out.release();
  if (c->s_h2d) cudaStreamDestroy(c->s_h2d);
  if (c->s_comp) cudaStreamDestroy(c->s_comp);
  if (c->s_d2h) cudaStreamDestroy(c->s_d2h);
  delete c;
  return VFI_OK;
}

int64_t vfi_launch_count(const vfi_ctx* c) { return c ? c->launches : 0; }

int vfi_set_batch(vfi_ctx* c, int batch) {
  if (!c || batch < 1 || batch > kMaxBatch) return fail(VFI_E_INVALID, "batch must be in [1,16]");
  c->batch = batch;
  return VFI_OK;
}

// Per-group device times of the forward schedule: CUDA events on the launching stream around each kernel group of every
// pass run while profiling is on (the groups and their ids are listed at span_begin).  Off by default: the event
// records break the dependent-launch chaining between groups, so the timed bench steps run without it.
int vfi_rife_profile(vfi_ctx* c, int enable) {
  if (!c) return fail(VFI_E_INVALID, "null ctx");
  CK(cudaSetDevice(c->device));
  CK(cudaDeviceSynchronize());
  for (auto& sp : c->prof_spans) {
    cudaEventDestroy(sp.e0);
    cudaEventDestroy(sp.e1);
  }
  c->prof_spans.clear();
  c->profile = enable != 0;
  return VFI_OK;
}

// Synchronises, then sums the recorded spans per group id: ids[i], total_ms[i], count[i] for up to `cap` groups; returns
// the number of groups through *n_out and clears the record.
int vfi_rife_profile_read(vfi_ctx* c, int32_t* ids, float* total_ms, int32_t* count, int cap, int* n_out) {
  if (!c || !ids || !total_ms || !count || !n_out || cap < 1) return fail(VFI_E_INVALID, "bad argument");
  CK(cudaSetDevice(c->device));
  CK(cudaDeviceSynchronize());
  int n = 0;
  for (auto& sp : c->prof_spans) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, sp.e0, sp.e1) != cudaSuccess) ms = 0.f;
    int k = 0;
    while (k < n && ids[k] != sp.id) ++k;
    if (k == n) {
      if (n == cap) continue;
      ids[n] = sp.id;
      total_ms[n] = 0.f;
      count[n] = 0;
      ++n;
    }
    total_ms[k] += ms;
    count[k] += 1;
    cudaEventDestroy(sp.e0);
    cudaEventDestroy(sp.e1);
  }
  c->prof_spans.clear();
  *n_out = n;
  return VFI_OK;
}

int vfi_sync(vfi_ctx* c) {
  if (!c) return fail(VFI_E_INVALID, "null ctx");
  CK(cudaSetDevice(c->device));
  CK(cudaDeviceSynchronize());
  return VFI_OK;
}

int vfi_rife46_load(vfi_ctx* c, const float* const* T, const int64_t* numel, int n_tensors, int operand_type) {
  return vfi_rife_load(c, 46, T, numel, n_tensors, operand_type);
}

int vfi_rife_load(vfi_ctx* c, int arch, const float* const* T, const int64_t* numel, int n_tensors, int operand_type) {
  if (!c || !T || !numel) return fail(VFI_E_INVALID, "null argument");
  if (arch != 46 && arch != 47 && arch != 417 && arch != 426)
    return fail(VFI_E_NOTIMPL,
                "RIFE arch must be 46 (rife46.pth), 47 (rife47/rife49.pth), 417 (rife417.pth) or 426 (rife426.pth)");
  if (n_tensors != (arch == 46 ? VFI_RIFE46_NUM_TENSORS : arch == 47 ? VFI_RIFE47_NUM_TENSORS
                    : arch == 417 ? VFI_RIFE417_NUM_TENSORS : VFI_RIFE426_NUM_TENSORS))
    return fail(VFI_E_INVALID,
                "wrong number of state_dict tensors for this RIFE arch (4.6: 120, 4.7: 124, 4.17: 128, 4.26: 158)");
  if (operand_type != OP_F16 && operand_type != OP_BF16) return fail(VFI_E_INVALID, "operand_type");
  CK(cudaSetDevice(c->device));
  free_weights(c);
  c->op_type = operand_type;
  c->arch = arch;
  int k = 0;
  auto expect = [&](int idx, int64_t want) { return numel[idx] == want; };
  const int nb = num_blocks(arch);
  const int nlast = arch == 426 ? 52 : 24;  // lastconv = ConvTranspose2d(c, 4*6 | 4*13, 4, 2, 1) - rife_arch.py:215-218, :230-233
  for (int b = 0; b < nb; ++b) {
    const int ch = kBlockC[b];
    const int cin = (arch == 426 ? kBlockCinReal426 : arch == 417 ? kBlockCinReal417 : arch == 47 ? kBlockCinReal47
                                                                                                  : kBlockCinReal)[b];
    if (!expect(k, (int64_t)(ch / 2) * cin * 9) || !expect(k + 1, ch / 2) || !expect(k + 2, (int64_t)ch * (ch / 2) * 9) ||
        !expect(k + 3, ch))
      return fail(VFI_E_INVALID, "conv0 tensor sizes do not match RIFE 4.6");
    TapConvLayer* Lb = c->layers[b];
    int r;
    if ((r = build_layer(c, Lb[LAYER_CONV00], LAYER_CONV00, arch != 46 ? 32 : 16, ch / 2,
                         conv2d(T[k], T[k + 1], cin, ch / 2))))
      return r;
    if ((r = build_layer(c, Lb[LAYER_CONV01], LAYER_CONV01, ch / 2, ch, conv2d(T[k + 2], T[k + 3], ch / 2, ch))))
      return r;
    k += 4;
    for (int j = 0; j < 8; ++j) {
      if (!expect(k, ch) || !expect(k + 1, (int64_t)ch * ch * 9) || !expect(k + 2, ch))
        return fail(VFI_E_INVALID, "convblock tensor sizes do not match RIFE 4.6");
      if ((r = build_layer(c, Lb[LAYER_RESCONV + j], LAYER_RESCONV, ch, ch, conv2d(T[k + 1], T[k + 2], ch, ch, T[k]))))
        return r;
      k += 3;
    }
    if (!expect(k, (int64_t)ch * nlast * 16) || !expect(k + 1, nlast))
      return fail(VFI_E_INVALID, "lastconv tensor sizes do not match this RIFE arch");
    // lastconv: column n = c5*16 + py*4 + px holds channel c5 < 5 at sub-pixel (py, px) of the cell's 4x4 patch
    const auto flow_col = [](int n) { return shuffled(n >> 4, (n >> 2) & 3, n & 3); };
    if ((r = build_layer(c, Lb[LAYER_LASTCONV], LAYER_LASTCONV, ch, 80,
                         conv_transpose(T[k], T[k + 1], ch, nlast, flow_col))))
      return r;
    // arch 4.26: channels 5..12 (rife_arch.py:230-233, :272), the 8 features handed to the next block: column
    // n = (py*4 + px)*8 + f, so 16 consecutive columns are two x-adjacent sub-pixels x 8 channels = 32 contiguous bytes
    // of the [B, 4H, 4W, 8] output (out_s2d = 2)
    const auto feat_col = [](int n) { return shuffled(5 + (n & 7), n >> 5, (n >> 3) & 3); };
    if (block_has_layer(arch, b, LAYER_LASTFEAT) &&
        (r = build_layer(c, Lb[LAYER_LASTFEAT], LAYER_LASTFEAT, ch, 128,
                         conv_transpose(T[k], T[k + 1], ch, nlast, feat_col))))
      return r;
    k += 2;
  }
  // Head cnn1, cnn2 (3x3 + LeakyReLU) and cnn3 (ConvTranspose2d(creal, cout, 4, 2, 1)) of arch 4.17 / 4.26 from their
  // weights and biases H[0..5], as tapconv layers on 32 channels, the kernel's smallest k-block (4.26's 16-channel layers
  // zero-padded).  cnn3's column n = (a*2 + b)*cout + oc: its NHWC output [Hh][Wh][4*cout] IS the space-to-depth form of
  // the feature map.
  auto build_head = [&](const float* const* H, int creal, int cout) {
    const auto col = [cout](int n) { return ConvTCol{n % cout, n / cout >> 1, n / cout & 1}; };
    int r;
    if ((r = build_layer(c, c->head[0], LAYER_HEAD_CONV, 32, 32, conv2d(H[0], H[1], creal, creal))) ||
        (r = build_layer(c, c->head[1], LAYER_HEAD_CONV, 32, 32, conv2d(H[2], H[3], creal, creal))))
      return r;
    return build_layer(c, c->head[2], LAYER_HEAD_DECONV, 32, 4 * cout, conv_transpose(H[4], H[5], creal, cout, col));
  };
  if (arch == 47) {  // encode = Conv2d(3,16,3,2,1) + ConvTranspose2d(16,4,4,2,1), fp32 on the CUDA cores
    const int64_t want[4] = {16 * 3 * 9, 16, 16 * 4 * 16, 4};
    for (int i = 0; i < 4; ++i) {
      if (numel[k + i] != want[i]) return fail(VFI_E_INVALID, "encode tensor sizes do not match RIFE 4.7");
      std::vector<float> h(T[k + i], T[k + i] + want[i]);
      int r;
      if ((r = upload(c, h, (void**)&c->enc[i]))) return r;
    }
    k += 4;
  }
  if (arch == 417) {  // encode = Head_417: cnn0 on the CUDA cores (fp32 weights), cnn1..cnn3 as tapconv layers
    const int64_t want[8] = {32 * 3 * 9, 32, 32 * 32 * 9, 32, 32 * 32 * 9, 32, 32 * 8 * 16, 8};
    for (int i = 0; i < 8; ++i)
      if (numel[k + i] != want[i]) return fail(VFI_E_INVALID, "encode tensor sizes do not match RIFE 4.17");
    int r;
    for (int i = 0; i < 2; ++i) {
      std::vector<float> h(T[k + i], T[k + i] + want[i]);
      if ((r = upload(c, h, (void**)&c->enc[i]))) return r;
    }
    if ((r = build_head(T + k + 2, 32, 8))) return r;
    k += 8;
  }
  if (arch == 426) {
    // encode = Head (rife_arch.py:378-395): the 16-channel layers run zero-padded to 32 channels - cnn0 on the CUDA
    // cores (fp32 weights, outputs 16..31 have zero weights and bias), cnn1..cnn3 as tapconv layers; cnn3's 4 output
    // channels x 2x2 sub-pixels = 16 columns
    const int64_t want[8] = {16 * 3 * 9, 16, 16 * 16 * 9, 16, 16 * 16 * 9, 16, 16 * 4 * 16, 4};
    for (int i = 0; i < 8; ++i)
      if (numel[k + i] != want[i]) return fail(VFI_E_INVALID, "encode tensor sizes do not match RIFE 4.26");
    int r;
    std::vector<float> w0(32 * 27, 0.f), b0(32, 0.f);
    std::copy(T[k], T[k] + 16 * 27, w0.begin());
    std::copy(T[k + 1], T[k + 1] + 16, b0.begin());
    if ((r = upload(c, w0, (void**)&c->enc[0]))) return r;
    if ((r = upload(c, b0, (void**)&c->enc[1]))) return r;
    if ((r = build_head(T + k + 2, 16, 4))) return r;
    k += 8;
  }
  c->loaded = true;
  return VFI_OK;
}

int vfi_rife46_forward(vfi_ctx* c, const float* frames, int n_frames, int H, int W, int C, const int32_t* f0,
                       const int32_t* f1, const float* t, int n_tasks, float scale_factor, float* out, void* stream) {
  if (!c || !frames || !out || (n_tasks > 0 && (!f0 || !f1 || !t))) return fail(VFI_E_INVALID, "null argument");
  if (!c->loaded) return fail(VFI_E_STATE, "vfi_rife46_load has not been called");
  if (C < 3 || H < 1 || W < 1 || n_frames < 1) return fail(VFI_E_INVALID, "bad frame shape");
  if (n_tasks == 0) return VFI_OK;
  int r;
  if ((r = check_tasks(f0, f1, n_tasks, 0, n_frames))) return r;
  CK(cudaSetDevice(c->device));
  Geometry g;
  if ((r = make_geometry(c->arch, H, W, scale_factor, &g))) return r;
  int lo = n_frames, hi = 0;
  for (int i = 0; i < n_tasks; ++i) {
    lo = std::min(lo, std::min(f0[i], f1[i]));
    hi = std::max(hi, std::max(f0[i], f1[i]) + 1);
  }
  const int B = std::min(c->batch, n_tasks);
  const Widths w = span_widths(c, g, B, n_tasks);
  if ((r = ensure_workspace(c, g, w, hi - lo))) return r;
  cudaStream_t st = (cudaStream_t)stream;
  LAUNCH(launch_prep_frames(frames + (size_t)lo * H * W * C, hi - lo, H, W, C, (float4*)c->imgs.p, (uint2*)c->imgs_h.p,
                            g.Hp, g.Wp, st));
  if (c->arch != 46) {  // encode head, once per source frame, in groups that fit the half-resolution scratch
    for (int f = 0; f < hi - lo; f += kMaxBatch) {
      const int cnt = std::min(kMaxBatch, hi - lo - f);
      if ((r = run_encode(c, g, f, cnt, st))) return r;
    }
  }
  std::vector<int32_t> w0(n_tasks), w1(n_tasks);  // frame indices into the prepared window
  for (int i = 0; i < n_tasks; ++i) {
    w0[i] = f0[i] - lo;
    w1[i] = f1[i] - lo;
  }
  for (int pos = 0; pos < n_tasks; pos += w.Bc) {
    const SpanTasks tk{w0.data() + pos, w1.data() + pos, t + pos};
    if ((r = forward_span(c, g, tk, std::min(w.Bc, n_tasks - pos), w, H, W, out + (size_t)pos * H * W * 3, st))) return r;
  }
  return VFI_OK;
}

int vfi_rife46_interpolate_host(vfi_ctx* c, const float* frames, int n_frames, int H, int W, int C, int frame_lo,
                                int frame_hi, const int32_t* f0, const int32_t* f1, const float* t,
                                const int32_t* out_slot, const int32_t* frame_slot, int n_tasks, float scale_factor,
                                float* out) {
  if (!c || !frames || (n_tasks > 0 && (!out || !f0 || !f1 || !t))) return fail(VFI_E_INVALID, "null argument");
  if (!c->loaded) return fail(VFI_E_STATE, "vfi_rife46_load has not been called");
  if (C < 3 || H < 1 || W < 1 || frame_lo < 0 || frame_hi > n_frames || frame_lo >= frame_hi)
    return fail(VFI_E_INVALID, "bad frame shape / range");
  if (n_tasks == 0) return VFI_OK;
  int r;
  if ((r = check_tasks(f0, f1, n_tasks, frame_lo, frame_hi))) return r;
  for (int i = 1; i < n_tasks; ++i)
    if (std::min(f0[i], f1[i]) < std::min(f0[i - 1], f1[i - 1]))
      return fail(VFI_E_INVALID, "tasks must be ordered by frame index (as RIFE_VFI.vfi builds them)");
  CK(cudaSetDevice(c->device));
  Geometry g;
  if ((r = make_geometry(c->arch, H, W, scale_factor, &g))) return r;
  const int nf = frame_hi - frame_lo;
  const int B = std::min(c->batch, n_tasks);
  const size_t frame_elems = (size_t)H * W * C, out_elems = (size_t)H * W * 3;
  const size_t frame_bytes = frame_elems * sizeof(float), out_bytes = out_elems * sizeof(float);
  // pass sizes: full batches in the middle; on a long clip the first and the last passes are small (1, 2, 4 pairs) so
  // that the exposed head (upload before the first pass) and tail (download after the last) are one or two frames
  // instead of a whole batch
  std::vector<int> pass_pos, pass_n;
  {
    const bool ramp = B >= 8 && n_tasks >= 4 * B;
    int pos = 0;
    if (ramp)
      for (int n = 1; n < B && n <= 4; n *= 2) { pass_pos.push_back(pos); pass_n.push_back(n); pos += n; }
    const int tail = ramp ? 7 : 0;
    while (n_tasks - pos - tail >= B || (!ramp && pos < n_tasks)) {
      const int n = std::min(B, n_tasks - pos);
      pass_pos.push_back(pos); pass_n.push_back(n); pos += n;
    }
    if (ramp) {
      const int rest = n_tasks - pos;  // 7 .. B + 6 pairs left: [rest - 3, 2, 1] or [rest - 7, 4, 2, 1]
      int tail_n[4], nt = 0;
      if (rest - 3 <= B) { tail_n[nt++] = rest - 3; } else { tail_n[nt++] = rest - 7; tail_n[nt++] = 4; }
      tail_n[nt++] = 2;
      tail_n[nt++] = 1;
      for (int i = 0; i < nt; ++i) { pass_pos.push_back(pos); pass_n.push_back(tail_n[i]); pos += tail_n[i]; }
    }
  }
  const int nb = (int)pass_n.size();

  // ---- the prepared-frame window is a RING: only frames some task references are uploaded, in order of first use, into
  // slot (upload counter % R).  R covers every frame from its upload to the pass after its last use, so that the slot a
  // pass's uploads overwrite was last read two passes ago (the copy stream runs one pass ahead of the compute stream
  // without waiting) - 2 B + 1 slots for consecutive pairs instead of the whole clip (tens of MB per 1080p frame: a clip
  // of a few thousand frames would not fit).  An event wait keeps any reuse correct regardless.
  std::vector<int> first_pass(nf, -1), last_pass(nf, -1), ctr(nf, -1), up_frames, up_end(nb, 0);
  for (int k = 0; k < nb; ++k)
    for (int i = 0; i < pass_n[k]; ++i)
      for (int f : {f0[pass_pos[k] + i] - frame_lo, f1[pass_pos[k] + i] - frame_lo}) {
        if (first_pass[f] < 0) first_pass[f] = k;
        last_pass[f] = k;
      }
  {
    std::vector<std::vector<int>> by_pass(nb);
    for (int f = 0; f < nf; ++f)
      if (first_pass[f] >= 0) by_pass[first_pass[f]].push_back(f);
    for (int k = 0; k < nb; ++k) {
      for (int f : by_pass[k]) {
        ctr[f] = (int)up_frames.size();
        up_frames.push_back(f);
      }
      up_end[k] = (int)up_frames.size();
    }
  }
  int R = 1;
  for (int f = 0; f < nf; ++f)
    if (ctr[f] >= 0) R = std::max(R, up_end[std::min(last_pass[f] + 1, nb - 1)] - ctr[f]);
  const Widths w{B, B, B, g.dense, -1};  // one pass per span: the upload ring sets the width
  if ((r = ensure_workspace(c, g, w, R))) return r;
  const int kRaw = 2 * kMaxBatch + 4;  // raw upload ring (frames), overwritten in stream order on the copy stream
  CK(c->raw.ensure((size_t)kRaw * frame_bytes));
  CK(c->outdev.ensure((size_t)2 * B * out_bytes));

  // ---- host staging.  Pinned caller memory is copied from / to directly.  Pageable memory (what a ComfyUI IMAGE
  // tensor is) goes through a small ring of pinned buffers: an uploader thread memcpy's frame by frame into it ahead of
  // the H2D copies, a downloader thread empties the D2H ring into the caller's tensor; each uses a few copy threads.
  // Pass-through frames (frame_slot): source frame f is also wanted unchanged (first 3 channels) at out + frame_slot[f].
  // The uploader thread makes that copy - and when `out` is page-locked the frame is then UPLOADED FROM THERE: the one
  // host copy the node contract needs anyway doubles as the staging copy (staging and pass-through as two separate host
  // copies can become the critical path on a few host cores).
  const bool stage_out = !is_pinned_host(out);
  auto via_out = [&](int f_abs) { return frame_slot != nullptr && !stage_out && frame_slot[f_abs] >= 0; };
  bool any_ring = false, any_pt = false;
  const bool src_pinned = is_pinned_host(frames + (size_t)frame_lo * frame_elems);
  for (int f : up_frames) any_ring = any_ring || (!src_pinned && !via_out(f + frame_lo));
  if (frame_slot)
    for (int f = frame_lo; f < frame_hi; ++f) any_pt = any_pt || frame_slot[f] >= 0;
  const bool stage_in = any_ring;
  const int copy_threads = env_int("VFI_COPY_THREADS", 12, 1, 32);
  const size_t ring_mb = (size_t)env_int("VFI_STAGE_MB", 384, 32, 8192);
  const int force_slots = env_int("VFI_STAGE_SLOTS", 0, 0, 64);  // tests: a ring far smaller than the clip
  const int NS = !stage_in ? 0 : force_slots ? force_slots : (int)std::max<size_t>(4, std::min<size_t>(32, (ring_mb << 20) / frame_bytes));
  const int ND = !stage_out ? 0 : force_slots ? force_slots : (int)std::max<size_t>(4, std::min<size_t>(48, (ring_mb << 20) / out_bytes));
  if (stage_in) CK(c->pin_in.ensure((size_t)NS * frame_bytes));
  if (stage_out) CK(c->pin_out.ensure((size_t)ND * out_bytes));

  std::vector<cudaEvent_t> ev_up(nb), ev_comp(nb), ev_down(nb), ev_in(NS), ev_out(ND);
  auto mk = [](std::vector<cudaEvent_t>& v) {
    for (auto& e : v)
      if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return false;
    return true;
  };
  for (auto& e : ev_up) e = nullptr;
  for (auto& e : ev_comp) e = nullptr;
  for (auto& e : ev_down) e = nullptr;
  for (auto& e : ev_in) e = nullptr;
  for (auto& e : ev_out) e = nullptr;
  if (!(mk(ev_up) && mk(ev_comp) && mk(ev_down) && mk(ev_in) && mk(ev_out))) return fail(VFI_E_CUDA, "cudaEventCreate failed");

  // shared progress counters of the three host threads (all under one mutex; the hand-offs are per frame, ~0.5 ms apart)
  std::mutex mu;
  std::condition_variable cv;
  bool abort_all = false;
  int staged = 0;        // uploader: frames [0, staged) of up_frames sit in the pinned ring
  int h2d_issued = 0;    // main: H2D copies [0, h2d_issued) have been enqueued (their ev_in is recorded)
  int d2h_issued = 0;    // main: D2H copies [0, d2h_issued) have been enqueued (their ev_out is recorded)
  int drained = 0;       // downloader: output frames [0, drained) have been copied to the caller's tensor
  std::vector<int> d2h_slot;  // output slot of D2H copy i
  d2h_slot.reserve(n_tasks);
  const int n_up = (int)up_frames.size();
  // upload u comes from: the caller's pinned tensor (-2), its pass-through slot in the pinned output (-1), or pinned
  // staging ring entry ring_of[u] >= 0 (a running count of ring uploads)
  std::vector<int> ring_of(n_up, -2);
  {
    int nr = 0;
    for (int u = 0; u < n_up; ++u) {
      const int fa = up_frames[u] + frame_lo;
      if (via_out(fa)) ring_of[u] = -1;
      else if (!src_pinned) ring_of[u] = nr++;
    }
  }
  const size_t px_frame = (size_t)H * W;

  // VFI_TRACE=1: where the host threads spent their time (stderr, one line per call)
  const bool trace = env_int("VFI_TRACE", 0, 0, 1) != 0;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto secs = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
    return std::chrono::duration<double>(b - a).count();
  };
  double up_copy_s = 0, up_wait_s = 0, dn_copy_s = 0, dn_wait_s = 0, main_wait_stage_s = 0, main_wait_drain_s = 0;
  const auto t_call = now();

  std::thread uploader, downloader;
  if (stage_in || any_pt)
    uploader = std::thread([&] {
      cudaSetDevice(c->device);
      CopyPool pool(copy_threads);
      std::vector<char> pt_done(nf, 0);
      for (int u = 0; u < n_up; ++u) {
        const auto tw = now();
        const int fa = up_frames[u] + frame_lo;
        const float* src = frames + (size_t)fa * frame_elems;
        const int ri = ring_of[u];
        if (ri >= NS && ri >= 0) {  // the H2D copy that last read this pinned slot has been enqueued, then: has completed
          {
            std::unique_lock<std::mutex> l(mu);
            cv.wait(l, [&] { return abort_all || h2d_issued > ri - NS; });
            if (abort_all) return;
          }
          cudaEventSynchronize(ev_in[ri % NS]);
        }
        const auto tc = now();
        if (ri >= 0) pool.copy((uint8_t*)c->pin_in.p + (size_t)(ri % NS) * frame_bytes, src, frame_bytes);
        if (frame_slot && frame_slot[fa] >= 0) {
          pool.copy_rgb(out + (size_t)frame_slot[fa] * out_elems, src, px_frame, C);
          pt_done[fa - frame_lo] = 1;
        }
        up_wait_s += secs(tw, tc);
        up_copy_s += secs(tc, now());
        {
          std::lock_guard<std::mutex> l(mu);
          staged = u + 1;
        }
        cv.notify_all();
      }
      if (frame_slot)  // pass-through frames no task references (skipped pairs)
        for (int f = frame_lo; f < frame_hi; ++f)
          if (frame_slot[f] >= 0 && !pt_done[f - frame_lo]) {
            const auto tc = now();
            pool.copy_rgb(out + (size_t)frame_slot[f] * out_elems, frames + (size_t)f * frame_elems, px_frame, C);
            up_copy_s += secs(tc, now());
          }
    });
  if (stage_out)
    downloader = std::thread([&] {
      cudaSetDevice(c->device);
      CopyPool pool(copy_threads);
      for (int v = 0; v < n_tasks; ++v) {
        int slot;
        const auto tw = now();
        {
          std::unique_lock<std::mutex> l(mu);
          cv.wait(l, [&] { return abort_all || d2h_issued > v; });
          if (abort_all) return;
          slot = d2h_slot[v];
        }
        cudaEventSynchronize(ev_out[v % ND]);
        const auto tc = now();
        pool.copy(out + (size_t)slot * out_elems, (const uint8_t*)c->pin_out.p + (size_t)(v % ND) * out_bytes, out_bytes);
        dn_wait_s += secs(tw, tc);
        dn_copy_s += secs(tc, now());
        {
          std::lock_guard<std::mutex> l(mu);
          drained = v + 1;
        }
        cv.notify_all();
      }
    });

  int rc = VFI_OK;
  auto body = [&]() -> int {
    int up = 0, down = 0;  // upload / download counters
    for (int k = 0; k < nb; ++k) {
      const int pos = pass_pos[k], n = pass_n[k];
      // H2D + prep of the frames this pass uses for the first time, on the copy stream
      while (up < up_end[k]) {
        const int slot = up % R, rslot = up % kRaw;
        int run = std::min(std::min(up_end[k] - up, kRaw / 2), std::min(R - slot, kRaw - rslot));
        // a run is prepared by one kernel launch: its frames must have the same channel stride (3 from the output's
        // pass-through slots, C otherwise)
        const bool run_rgb = ring_of[up] == -1;
        for (int j = 1; j < run; ++j)
          if ((ring_of[up + j] == -1) != run_rgb) run = j;
        const size_t run_elems = run_rgb ? out_elems : frame_elems;
        for (int j = 0; j < run; ++j) {
          const int u = up + j;
          if (u >= R) CK(cudaStreamWaitEvent(c->s_h2d, ev_comp[last_pass[up_frames[u - R]]], 0));  // slot's last reader
          const int fa = up_frames[u] + frame_lo;
          const int ri = ring_of[u];
          const float* src = frames + (size_t)fa * frame_elems;
          if (ri != -2) {  // staged by the uploader thread
            const auto tw = now();
            std::unique_lock<std::mutex> l(mu);
            cv.wait(l, [&] { return staged > u; });
            src = (ri == -1) ? out + (size_t)frame_slot[fa] * out_elems
                             : (const float*)((const uint8_t*)c->pin_in.p + (size_t)(ri % NS) * frame_bytes);
            main_wait_stage_s += secs(tw, now());
          }
          CK(cudaMemcpyAsync((float*)c->raw.p + (size_t)rslot * frame_elems + (size_t)j * run_elems, src,
                             run_elems * sizeof(float), cudaMemcpyHostToDevice, c->s_h2d));
          if (ri >= 0) {
            CK(cudaEventRecord(ev_in[ri % NS], c->s_h2d));
            {
              std::lock_guard<std::mutex> l(mu);
              h2d_issued = ri + 1;
            }
            cv.notify_all();
          }
        }
        const size_t px = (size_t)g.Hp * g.Wp;
        LAUNCH(launch_prep_frames((float*)c->raw.p + (size_t)rslot * frame_elems, run, H, W, run_rgb ? 3 : C,
                                  (float4*)c->imgs.p + (size_t)slot * px, (uint2*)c->imgs_h.p + (size_t)slot * px, g.Hp, g.Wp,
                                  c->s_h2d));
        if (c->arch != 46) {
          const int r3 = run_encode(c, g, slot, run, c->s_h2d);
          if (r3) return r3;
        }
        up += run;
      }
      CK(cudaEventRecord(ev_up[k], c->s_h2d));
      CK(cudaStreamWaitEvent(c->s_comp, ev_up[k], 0));
      if (k >= 2) CK(cudaStreamWaitEvent(c->s_comp, ev_down[k - 2], 0));  // output slot free again
      int32_t w0[kMaxBatch], w1[kMaxBatch];  // ring slots of the pass's frames
      for (int i = 0; i < n; ++i) {
        w0[i] = ctr[f0[pos + i] - frame_lo] % R;
        w1[i] = ctr[f1[pos + i] - frame_lo] % R;
      }
      float* od = (float*)c->outdev.p + (size_t)(k & 1) * B * out_elems;
      int r2 = forward_span(c, g, SpanTasks{w0, w1, t + pos}, n, w, H, W, od, c->s_comp);
      if (r2) return r2;
      CK(cudaEventRecord(ev_comp[k], c->s_comp));
      CK(cudaStreamWaitEvent(c->s_d2h, ev_comp[k], 0));
      if (stage_out) {
        for (int i = 0; i < n; ++i, ++down) {
          {  // the downloader has emptied the pinned slot this copy lands in
            const auto tw = now();
            std::unique_lock<std::mutex> l(mu);
            cv.wait(l, [&] { return drained > down - ND; });
            main_wait_drain_s += secs(tw, now());
          }
          CK(cudaMemcpyAsync((uint8_t*)c->pin_out.p + (size_t)(down % ND) * out_bytes, od + (size_t)i * out_elems, out_bytes,
                             cudaMemcpyDeviceToHost, c->s_d2h));
          CK(cudaEventRecord(ev_out[down % ND], c->s_d2h));
          {
            std::lock_guard<std::mutex> l(mu);
            d2h_slot.push_back(out_slot ? out_slot[pos + i] : pos + i);
            d2h_issued = down + 1;
          }
          cv.notify_all();
        }
      } else if (!out_slot) {
        CK(cudaMemcpyAsync(out + (size_t)pos * out_elems, od, (size_t)n * out_bytes, cudaMemcpyDeviceToHost, c->s_d2h));
      } else {
        for (int i = 0; i < n; ++i)
          CK(cudaMemcpyAsync(out + (size_t)out_slot[pos + i] * out_elems, od + (size_t)i * out_elems, out_bytes,
                             cudaMemcpyDeviceToHost, c->s_d2h));
      }
      CK(cudaEventRecord(ev_down[k], c->s_d2h));
    }
    CK(cudaStreamSynchronize(c->s_d2h));
    CK(cudaStreamSynchronize(c->s_comp));
    CK(cudaStreamSynchronize(c->s_h2d));
    return VFI_OK;
  };
  rc = body();
  if (rc != VFI_OK) {
    {
      std::lock_guard<std::mutex> l(mu);
      abort_all = true;
    }
    cv.notify_all();
    cudaDeviceSynchronize();
  }
  if (uploader.joinable()) uploader.join();
  if (downloader.joinable()) downloader.join();
  if (trace)
    fprintf(stderr,
            "vfi trace: interpolate_host dev %d  %d tasks  %d uploads (ring %d)  total %.1f ms | stage_in=%d NS=%d copy %.1f ms "
            "wait %.1f ms | stage_out=%d ND=%d copy %.1f ms wait %.1f ms | main waited %.1f ms for staging, %.1f ms for draining\n",
            c->device, n_tasks, n_up, R, 1e3 * secs(t_call, now()), (int)stage_in, NS, 1e3 * up_copy_s, 1e3 * up_wait_s, (int)stage_out,
            ND, 1e3 * dn_copy_s, 1e3 * dn_wait_s, 1e3 * main_wait_stage_s, 1e3 * main_wait_drain_s);
  for (auto* v : {&ev_up, &ev_comp, &ev_down, &ev_in, &ev_out})
    for (auto e : *v)
      if (e) cudaEventDestroy(e);
  return rc;
}

// Host utility of the node: copy source frame i (first 3 of C channels) to out + slot[i] * H * W * 3 for every i with
// slot[i] >= 0, with `threads` copy threads - the pass-through frames of the output clip (rife/__init__.py:227-231 does a
// torch.cat of per-frame tensors).  Plain host memory on both sides; runs beside vfi_rife46_interpolate_host.
int vfi_host_copy_frames(const float* frames, int n_frames, int H, int W, int C, const int32_t* slot, float* out, int threads) {
  if (!frames || !slot || !out || n_frames < 1 || H < 1 || W < 1 || C < 3) return fail(VFI_E_INVALID, "bad argument");
  if (threads < 1) threads = 1;
  if (threads > 64) threads = 64;
  const size_t px = (size_t)H * W;
  std::vector<std::thread> th;
  std::atomic<int> next{0};
  for (int k = 0; k < threads; ++k)
    th.emplace_back([&] {
      // work items: (frame, quarter of the frame) so that a handful of frames still spreads over all threads
      for (;;) {
        const int item = next.fetch_add(1);
        const int f = item >> 2, q = item & 3;
        if (f >= n_frames) return;
        if (slot[f] < 0) continue;
        const size_t lo = px * q / 4, hi = px * (q + 1) / 4;
        const float* s = frames + (size_t)f * px * C;
        float* d = out + (size_t)slot[f] * px * 3;
        if (C == 3) {
          stream_copy(d + lo * 3, s + lo * 3, (hi - lo) * 3 * sizeof(float));
        } else {
          for (size_t i = lo; i < hi; ++i) {
            d[i * 3 + 0] = s[i * C + 0];
            d[i * 3 + 1] = s[i * C + 1];
            d[i * 3 + 2] = s[i * C + 2];
          }
        }
      }
    });
  for (auto& t : th) t.join();
  return VFI_OK;
}

int vfi_warp_bilinear_border(vfi_ctx* c, const float* img, const float* flow, float* out, int B, int H, int W, int C,
                             void* stream) {
  if (!c || !img || !flow || !out || B < 1 || H < 1 || W < 1 || C < 1) return fail(VFI_E_INVALID, "bad argument");
  CK(cudaSetDevice(c->device));
  LAUNCH(launch_warp(img, flow, out, B, H, W, C, (cudaStream_t)stream));
  return VFI_OK;
}

int vfi_softsplat_sum(vfi_ctx* c, const float* in, const float* flow, float* out, int N, int C, int H, int W,
                      void* stream) {
  if (!c || !in || !flow || !out || N < 1 || C < 1 || H < 1 || W < 1) return fail(VFI_E_INVALID, "bad argument");
  CK(cudaSetDevice(c->device));
  LAUNCH(launch_softsplat_sum(in, flow, out, N, C, H, W, (cudaStream_t)stream));
  return VFI_OK;
}

int vfi_softsplat_weighted(vfi_ctx* c, const float* in, const float* flow, const float* metric, int mode, int eps, float* out,
                           float* norm, int N, int C, int H, int W, void* stream) {
  if (!c || !in || !flow || !out || !norm || N < 1 || C < 1 || H < 1 || W < 1) return fail(VFI_E_INVALID, "bad argument");
  if (mode < 0 || mode > 2 || eps < 0 || eps > 2 || (mode != 0 && !metric)) return fail(VFI_E_INVALID, "softsplat mode / eps / metric");
  CK(cudaSetDevice(c->device));
  // default: the channel-last form (16-byte vector atomics); VFI_SPLAT_NHWC=0: the NCHW scalar-atomic kernels (A/B runs)
  static const bool nhwc = [] {
    const char* e = std::getenv("VFI_SPLAT_NHWC");
    return !(e && e[0] == '0');
  }();
  if (nhwc && N <= 65535) {
    const size_t fl = ops_scratch_floats(N, C, H, W) * sizeof(float);
    CK(c->ops_a.ensure(fl));
    CK(c->ops_b.ensure(fl));
    CK(launch_softsplat_weighted_nhwc(in, flow, metric, mode, eps, out, norm, (float*)c->ops_a.p, (float*)c->ops_b.p, N, C, H, W,
                                      static_cast<cudaStream_t>(stream)));
    c->launches += 3;
    return VFI_OK;
  }
  CK(launch_softsplat_weighted(in, flow, metric, mode, eps, out, norm, N, C, H, W, static_cast<cudaStream_t>(stream)));
  c->launches += 2;
  return VFI_OK;
}

int vfi_costvol_l1(vfi_ctx* c, const float* one, const float* two, float* out, int N, int C, int H, int W,
                   void* stream) {
  if (!c || !one || !two || !out || N < 1 || C < 1 || H < 1 || W < 1) return fail(VFI_E_INVALID, "bad argument");
  CK(cudaSetDevice(c->device));
  // VFI_VOLUME_WARP=1: the warp-per-pixel channel-last form (shuffle reduction over the channels).  Each displacement
  // re-reads its channel vector through L1, 81 times per pixel, so the shared-memory tiled kernel stays the default and
  // this form is kept for comparison.
  static const bool warp_form = [] {
    const char* e = std::getenv("VFI_VOLUME_WARP");
    return e && e[0] == '1';
  }();
  if (warp_form && N <= 65535 && H <= 65535) {
    const size_t fl = ops_scratch_floats(N, C, H, W) * sizeof(float);
    CK(c->ops_a.ensure(fl));
    CK(c->ops_b.ensure(fl));
    CK(launch_volume81_warp(false, one, two, out, (float*)c->ops_a.p, (float*)c->ops_b.p, N, C, H, W, (cudaStream_t)stream));
    c->launches += 3;
    return VFI_OK;
  }
  LAUNCH(launch_volume81(false, one, two, out, N, C, H, W, (cudaStream_t)stream));
  return VFI_OK;
}

int vfi_corr_dot(vfi_ctx* c, const float* first, const float* second, float* out, int N, int C, int H, int W,
                 void* stream) {
  if (!c || !first || !second || !out || N < 1 || C < 1 || H < 1 || W < 1) return fail(VFI_E_INVALID, "bad argument");
  CK(cudaSetDevice(c->device));
  // VFI_VOLUME_WARP=1: the warp-per-pixel channel-last form (shuffle reduction over the channels).  Each displacement
  // re-reads its channel vector through L1, 81 times per pixel, so the shared-memory tiled kernel stays the default and
  // this form is kept for comparison.
  static const bool warp_form = [] {
    const char* e = std::getenv("VFI_VOLUME_WARP");
    return e && e[0] == '1';
  }();
  if (warp_form && N <= 65535 && H <= 65535) {
    const size_t fl = ops_scratch_floats(N, C, H, W) * sizeof(float);
    CK(c->ops_a.ensure(fl));
    CK(c->ops_b.ensure(fl));
    CK(launch_volume81_warp(true, first, second, out, (float*)c->ops_a.p, (float*)c->ops_b.p, N, C, H, W, (cudaStream_t)stream));
    c->launches += 3;
    return VFI_OK;
  }
  LAUNCH(launch_volume81(true, first, second, out, N, C, H, W, (cudaStream_t)stream));
  return VFI_OK;
}

int vfi_sepconv(vfi_ctx* c, const float* in, const float* ver, const float* hor, float* out, int N, int C, int H,
                int W, int Kv, int Kh, void* stream) {
  if (!c || !in || !ver || !hor || !out || N < 1 || C < 1 || H < 1 || W < 1 || Kv < 1 || Kh < 1)
    return fail(VFI_E_INVALID, "bad argument");
  CK(cudaSetDevice(c->device));
  LAUNCH(launch_sepconv(in, ver, hor, out, N, C, H, W, Kv, Kh, (cudaStream_t)stream));
  return VFI_OK;
}

int vfi_adacof(vfi_ctx* c, const float* in, const float* weight, const float* offset_i, const float* offset_j, float* out, int N,
               int C, int Hin, int Win, int F, int dilation, int Ho, int Wo, void* stream) {
  if (!c || !in || !weight || !offset_i || !offset_j || !out || N < 1 || C < 1 || Ho < 1 || Wo < 1)
    return fail(VFI_E_INVALID, "bad argument");
  if (F < 1 || dilation < 1 || Hin - ((F - 1) * dilation + 1) != Ho - 1 || Win - ((F - 1) * dilation + 1) != Wo - 1)
    return fail(VFI_E_INVALID, "adacof: input size must be output size + (F - 1) * dilation (adacof.py:274-279)");
  CK(cudaSetDevice(c->device));
  CK(launch_adacof(in, weight, offset_i, offset_j, out, N, C, Hin, Win, F, dilation, Ho, Wo, static_cast<cudaStream_t>(stream)));
  c->launches += 1;
  return VFI_OK;
}

int vfi_edt_pass(vfi_ctx* c, const float* data, float* out, int bs, int h, int w, float diam2, void* stream) {
  if (!c || !data || !out || bs < 1 || h < 1 || w < 1) return fail(VFI_E_INVALID, "bad argument");
  CK(cudaSetDevice(c->device));
  CK(launch_edt_pass(data, out, bs, h, w, diam2, static_cast<cudaStream_t>(stream)));
  c->launches += 1;
  return VFI_OK;
}

int vfi_rife46_debug_layer(vfi_ctx* c, int block, int layer, const void* in, void* out, void* out_mask, int B, int H,
                           int W, int impl, void* stream) {
  if (!c || block < 0 || layer < 0 || !in || !out) return fail(VFI_E_INVALID, "bad argument");
  if (!c->loaded) return fail(VFI_E_STATE, "vfi_rife46_load has not been called");
  if (!block_has_layer(c->arch, block, layer)) return fail(VFI_E_INVALID, "no such block / layer in the loaded arch");
  if (impl != TAPCONV_PLANNED && impl != TAPCONV_CHECKER && impl != TAPCONV_CELL_MAJOR)
    return fail(VFI_E_INVALID, "impl must be 0 (tensor cores), 1 (checker) or 2 (tensor cores, cell-major MMAs)");
  CK(cudaSetDevice(c->device));
  const TapConvLayer& L = c->layers[block][layer];
  if (layer == LAYER_LASTCONV) {
    if (!out_mask) return fail(VFI_E_INVALID, "lastconv needs out_mask");
    LAUNCH(launch_tapconv(L, c->op_type, in, nullptr, (float4*)out, (float*)out_mask, B, H, W, c->num_sms, impl,
                          (cudaStream_t)stream));
  } else {
    LAUNCH(launch_tapconv(L, c->op_type, in, out, nullptr, nullptr, B, H, W, c->num_sms, impl,
                          (cudaStream_t)stream));
  }
  return VFI_OK;
}

int vfi_rife46_debug_conv0_fused(vfi_ctx* c, int block, const void* in, void* out, int B, int H, int W, void* stream) {
  if (!c || block < 0 || !in || !out) return fail(VFI_E_INVALID, "bad argument");
  if (!c->loaded) return fail(VFI_E_STATE, "vfi_rife46_load has not been called");
  if (!block_has_layer(c->arch, block, LAYER_CONV01)) return fail(VFI_E_INVALID, "no such block in the loaded arch");
  const TapConvLayer& L0 = c->layers[block][LAYER_CONV00];
  const TapConvLayer& L1 = c->layers[block][LAYER_CONV01];
  if (c->arch != 46 || conv0_fused_plan(L0, L1, c->op_type, nullptr, nullptr, nullptr) < 1)
    return fail(VFI_E_INVALID, "this block's conv0.0 / conv0.1 do not run as one launch");
  CK(cudaSetDevice(c->device));
  LAUNCH(launch_conv0_fused(L0, L1, c->op_type, in, nullptr, out, B, H, W, c->num_sms, (cudaStream_t)stream));
  return VFI_OK;
}

int vfi_rife46_debug_unfused_conv0(vfi_ctx* c, int unfused) {
  if (!c) return fail(VFI_E_INVALID, "null context");
  c->conv0_unfused = unfused != 0;
  return VFI_OK;
}

int vfi_rife46_debug_state(vfi_ctx* c, float* flow4_out, float* mask_out, int batch, int* Hp, int* Wp) {
  if (!c || !Hp || !Wp) return fail(VFI_E_INVALID, "null argument");
  CK(cudaSetDevice(c->device));
  CK(cudaDeviceSynchronize());
  *Hp = c->ws_Hp;
  *Wp = c->ws_Wp;
  if (!flow4_out && !mask_out) return VFI_OK;
  if (batch < 1 || batch > c->ws_B) return fail(VFI_E_INVALID, "batch larger than the last pass");
  // the full-resolution flow is implicit on the product path; materialise it for the caller
  const size_t n = (size_t)batch * c->ws_Hp * c->ws_Wp;
  CK(c->dbgF.ensure(n * sizeof(float4)));
  CK(c->dbgM.ensure(n * sizeof(float)));
  if (c->last_lo >= c->last_fs.n) {  // every level already folded into the dense planes (up-scaled last blocks)
    CK(cudaMemcpy(c->dbgF.p, c->last_F, n * sizeof(float4), cudaMemcpyDeviceToDevice));
    CK(cudaMemcpy(c->dbgM.p, c->last_M, n * sizeof(float), cudaMemcpyDeviceToDevice));
  } else {
    LAUNCH(launch_materialize(c->last_fs, c->last_lo, c->last_have_base ? c->last_F : nullptr,
                              c->last_have_base ? c->last_M : nullptr, (float4*)c->dbgF.p,
                              (float*)c->dbgM.p, batch, c->ws_Hp, c->ws_Wp, 0));
  }
  CK(cudaDeviceSynchronize());
  if (flow4_out) CK(cudaMemcpy(flow4_out, c->dbgF.p, n * sizeof(float4), cudaMemcpyDeviceToDevice));
  if (mask_out) CK(cudaMemcpy(mask_out, c->dbgM.p, n * sizeof(float), cudaMemcpyDeviceToDevice));
  return VFI_OK;
}

int vfi_rife46_layer_plan(vfi_ctx* c, int block, int layer, int* stages, int* n_cta, int* nsplit, int* smem_bytes,
                          int64_t* macs_per_cell, int* cmajor, int* wstream) {
  if (!c || block < 0 || layer < 0) return fail(VFI_E_INVALID, "bad argument");
  if (!c->loaded) return fail(VFI_E_STATE, "vfi_rife46_load has not been called");
  if (!block_has_layer(c->arch, block, layer)) return fail(VFI_E_INVALID, "no such block / layer in the loaded arch");
  const TapConvLayer& L = c->layers[block][layer];
  TapConvParams p{};
  const int st = tapconv_plan(L, &p);
  if (stages) *stages = st;
  if (n_cta) *n_cta = L.n_cta;
  if (nsplit) *nsplit = L.nsplit;
  if (smem_bytes) *smem_bytes = (int)p.smem_bytes;
  // (a streamed 3x3 layer may issue K=16 steps with zero weights after its 9 x cin products per output: c = 96 two)
  if (macs_per_cell) *macs_per_cell = (int64_t)(L.wstream ? 9 * L.cin : L.ktotal16 * 16) * L.n_total;
  if (cmajor) *cmajor = p.cmajor;
  if (wstream) *wstream = p.wstream;
  return VFI_OK;
}

int vfi_rife46_conv0_plan(vfi_ctx* c, int block, int32_t* info, int cap) {
  if (!c || block < 0 || (!info && cap > 0)) return fail(VFI_E_INVALID, "bad argument");
  if (!c->loaded) return fail(VFI_E_STATE, "vfi_rife46_load has not been called");
  if (!block_has_layer(c->arch, block, LAYER_CONV01)) return fail(VFI_E_INVALID, "no such block in the loaded arch");
  int32_t v[5] = {0, 0, 0, 0, 0};
  if (c->arch == 46) {
    int smem = 0, regs = 0, local = 0;
    v[1] = conv0_fused_plan(c->layers[block][LAYER_CONV00], c->layers[block][LAYER_CONV01], c->op_type, &smem, &regs,
                            &local);
    v[0] = v[1] > 0 ? 1 : 0;
    v[2] = smem;
    v[3] = regs;
    v[4] = local;
  }
  for (int k = 0; k < cap && k < 5; ++k) info[k] = v[k];
  return VFI_OK;
}

}  // extern "C"
