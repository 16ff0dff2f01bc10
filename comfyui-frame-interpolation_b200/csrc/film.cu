// FILM (film_net) on H100: weight repacking, workspace, the forward schedule and its C ABI (include/vfi_b200.h).
// SURVEY.md section 8 row a10.  Reference: vfi_models/film/film_arch.py, Interpolator.debug_forward :401-456.
//
// Forward schedule for B frame pairs (images are indexed k*B + pair, k = 0 first frame, 1 second frame; H_l = H >> l):
//   gather_rgb, 6 x pool_rgb                  image pyramids, 7 levels                              :655-674
//   7 sub-trees (shared weights)              conv_rgb / streamconv / pool16; the second conv of sub-level j of image
//                                             level i writes channel slice [0|64|192|448] of feat[i+j]   :102-121,:133-163
//   2 directions x 7 levels, coarse to fine   flow_up -> warp16 -> 4 x streamconv (conv 0 reads cat(feat_a, warped_b)
//                                             from two tensors) -> flow_head (v = residual + up)          :567-616
//   5 levels                                  aligned[l] = [warp(feat0, bwd/2) | warp(feat1, fwd/2) | misc64]   :425-447
//   4 fusion levels, coarse to fine           nearest16 -> streamconv 2x2 -> streamconv 3x3 on cat(aligned, net) ->
//                                             streamconv 3x3                                               :258-296
//   out_rgb                                   1x1 conv 64 -> 3 (+ the node's clamp, film/__init__.py:38)
// Channel layouts in HBM differ from the reference's concatenation order (64-channel alignment); the weight packer
// below maps every padded input channel to its reference channel (or to a zero weight).
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

constexpr int kLevels = 7, kFuseLevels = 5, kSub = 4;
const int kFeatC[kLevels] = {64, 192, 448, 960, 960, 960, 960};  // cascaded feature channels per level (film_arch.py:155-163)
const int kSliceOff[kSub] = {0, 64, 192, 448};                   // slice of sub-level j inside a feature level
const int kFlowNF[4] = {32, 64, 128, 256};                       // flow_filters (film_arch.py:386); index 3 = shared predictor

struct Buf {
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

struct FilmState {
  int op_type = OP_F16;
  bool loaded = false;
  bool use_ref = false;  // debug: every conv through the CUDA-core checker (vfi_film_debug_set_ref)
  std::vector<void*> allocs;
  // ---- layers
  float* rgb_w = nullptr;  // extract.convs.0.0: Conv2d(3, 64, 3) on the CUDA cores
  float* rgb_b = nullptr;
  StreamConvLayer ext[kSub][2];   // ext[j][0] (j >= 1): 64<<(j-1) -> 64<<j; ext[j][1]: 64<<j -> 64<<j
  StreamConvLayer flow[4][4];     // [predictor: 0..2 = levels 0..2, 3 = shared (levels 3..6)][conv 0..2 (3x3), 3 (1x1)]
  float* head_w[4] = {nullptr, nullptr, nullptr, nullptr};  // Conv2d(nf/2, 2, 1) per predictor
  float* head_b[4] = {nullptr, nullptr, nullptr, nullptr};
  StreamConvLayer fuse[4][3];     // [k: coarse to fine][2x2, 3x3 on cat, 3x3]
  float* out_w = nullptr;
  float* out_b = nullptr;
  // ---- workspace
  Buf img[kLevels], feat[kLevels], v[2][kLevels], aligned[kFuseLevels];
  Buf tmpA, tmpB, vup, wb, t0, t1, t3, upbuf, n0, n1, n2;
  int64_t macs = 0;  // tensor-core MACs of the last forward (real channels, bench.py)
  int last_B = 0;    // pairs and level sizes of the last forward (vfi_film_debug_state)
  int last_H[kLevels] = {}, last_W[kLevels] = {};
};

void film_destroy(FilmState* f) {
  if (!f) return;
  for (void* p : f->allocs) cudaFree(p);
  for (int l = 0; l < kLevels; ++l) {
    f->img[l].release();
    f->feat[l].release();
    f->v[0][l].release();
    f->v[1][l].release();
  }
  for (int l = 0; l < kFuseLevels; ++l) f->aligned[l].release();
  for (Buf* b : {&f->tmpA, &f->tmpB, &f->vup, &f->wb, &f->t0, &f->t1, &f->t3, &f->upbuf, &f->n0, &f->n1, &f->n2})
    b->release();
  delete f;
}

namespace {

#define FCK(call)                                                            \
  do {                                                                       \
    cudaError_t _e = (call);                                                 \
    if (_e != cudaSuccess) {                                                 \
      set_error(std::string(#call) + ": " + cudaGetErrorString(_e));         \
      return VFI_E_CUDA;                                                     \
    }                                                                        \
  } while (0)

int ffail(int code, const std::string& msg) {
  set_error(msg);
  return code;
}

template <class T>
int fupload(FilmState* f, const T* h, size_t n, void** dptr) {
  void* d = nullptr;
  FCK(cudaMalloc(&d, n * sizeof(T)));
  f->allocs.push_back(d);
  FCK(cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice));
  *dptr = d;
  return VFI_OK;
}

// Packs a PyTorch Conv2d weight [cout][cin][k][k] into streamconv's operand layout (host only, no CUDA calls):
// [split][k-block][tap][n_cta rows][64 channels, 16-byte chunks XOR (row & 7)], zero where the padded input channel
// has no reference channel (kmap[j] = -1) or the padded output column no filter (n >= cout).
int pack_conv(int op_type, int ksize, int c0, int c1, int n_total, const float* w, int cout, int cin,
              const std::vector<int>& kmap, std::vector<uint16_t>* out, StreamConvParams* plan) {
  if ((int)kmap.size() != c0 + c1) return ffail(VFI_E_INVALID, "film: channel map size");
  for (int ci : kmap)
    if (ci >= cin) return ffail(VFI_E_INVALID, "film: channel map out of range");
  const int ntaps = ksize * ksize;
  StreamConvLayer L;
  L.ksize = ksize;
  L.c0 = c0;
  L.c1 = c1;
  L.n_total = n_total;
  if (!pack_streamconv(L, op_type, [&](int n, int tap, int j) -> float {
        const int ci = kmap[j];  // tap = ky * k + kx, PyTorch weight [n][ci][ky][kx]
        return (n < cout && ci >= 0) ? w[((size_t)n * cin + ci) * ntaps + tap] : 0.f;
      }, out, plan))
    return ffail(VFI_E_INVALID, "film: layer shape not supported by streamconv");
  return VFI_OK;
}

// Builds one streamconv layer (packed weights + bias on the device) from a PyTorch Conv2d weight and bias.
// kmap[j] = reference input channel of padded input channel j (or -1: zero weight); size c0 + c1.
int build_conv(FilmState* f, StreamConvLayer& L, int ksize, int c0, int c1, int n_total, int act, const float* w,
               const float* bias, int cout, int cin, const std::vector<int>& kmap) {
  L = StreamConvLayer{};
  L.ksize = ksize;
  L.c0 = c0;
  L.c1 = c1;
  L.n_total = n_total;
  L.act = act;
  StreamConvParams p{};
  std::vector<uint16_t> pk;
  int rc = pack_conv(f->op_type, ksize, c0, c1, n_total, w, cout, cin, kmap, &pk, &p);
  if (rc) return rc;
  std::vector<float> sh(n_total, 0.f);
  for (int n = 0; n < cout && n < n_total; ++n) sh[n] = bias[n];
  rc = fupload(f, pk.data(), pk.size(), &L.w);
  if (rc) return rc;
  void* d = nullptr;
  rc = fupload(f, sh.data(), sh.size(), &d);
  L.shift = static_cast<float*>(d);
  return rc;
}

std::vector<int> identity_map(int real, int padded) {
  std::vector<int> m(padded, -1);
  for (int i = 0; i < real; ++i) m[i] = i;
  return m;
}

// our aligned-level layout [wfeat0 C | wfeat1 C | misc 64] -> reference order
// [wimg0 3, wfeat0 C, wimg1 3, wfeat1 C, bwd 2, fwd 2] (film_arch.py:431-447)
std::vector<int> aligned_map(int C) {
  std::vector<int> m(2 * C + 64, -1);
  for (int j = 0; j < C; ++j) {
    m[j] = 3 + j;
    m[C + j] = 3 + C + 3 + j;
  }
  for (int j = 0; j < 3; ++j) {
    m[2 * C + j] = j;
    m[2 * C + 3 + j] = 3 + C + j;
  }
  m[2 * C + 6] = 2 * C + 6;
  m[2 * C + 7] = 2 * C + 7;
  m[2 * C + 8] = 2 * C + 8;
  m[2 * C + 9] = 2 * C + 9;
  return m;
}

struct Dims {
  int H[kLevels], W[kLevels];
  size_t px(int l) const { return (size_t)H[l] * W[l]; }
};

int ensure_workspace(FilmState* f, const Dims& d, int B) {
  const size_t px0 = d.px(0);
  for (int l = 0; l < kLevels; ++l) {
    FCK(f->img[l].ensure((size_t)2 * B * d.px(l) * 3 * 4));
    FCK(f->feat[l].ensure((size_t)2 * B * d.px(l) * kFeatC[l] * 2));
    FCK(f->v[0][l].ensure((size_t)B * d.px(l) * 2 * 4));
    FCK(f->v[1][l].ensure((size_t)B * d.px(l) * 2 * 4));
  }
  for (int l = 0; l < kFuseLevels; ++l) FCK(f->aligned[l].ensure((size_t)B * d.px(l) * (2 * kFeatC[l] + 64) * 2));
  FCK(f->tmpA.ensure((size_t)2 * B * px0 * 64 * 2));
  FCK(f->tmpB.ensure((size_t)2 * B * d.px(1) * 64 * 2 + 256));
  FCK(f->vup.ensure((size_t)B * px0 * 2 * 4));
  size_t wb = 0, up = 0;
  for (int l = 0; l < kLevels; ++l) wb = std::max(wb, (size_t)B * d.px(l) * kFeatC[l] * 2);
  FCK(f->wb.ensure(wb));
  FCK(f->t0.ensure((size_t)B * px0 * 64 * 2));
  FCK(f->t1.ensure((size_t)B * px0 * 64 * 2));
  FCK(f->t3.ensure((size_t)B * px0 * 16 * 2));
  const int netc[4] = {2 * 960 + 64, 512, 256, 128};
  for (int k = 0; k < 4; ++k) up = std::max(up, (size_t)B * d.px(3 - k) * netc[k] * 2);
  FCK(f->upbuf.ensure(up));
  FCK(f->n0.ensure((size_t)B * px0 * 64 * 2));
  FCK(f->n1.ensure((size_t)B * px0 * 64 * 2));
  FCK(f->n2.ensure((size_t)B * px0 * 64 * 2));
  return VFI_OK;
}

struct Runner {
  vfi_ctx* c;
  FilmState* f;
  CtxInfo ci;
  cudaStream_t st;
  int launches = 0;
  int conv(const StreamConvLayer& L, const void* s0, int p0, const void* s1, int p1, void* out, int op, int B, int H, int W,
           int64_t real_macs_per_px) {
    const cudaError_t e = launch_streamconv(L, f->op_type, s0, p0, s1, p1, out, op, B, H, W, ci.num_sms, f->use_ref, st);
    ++launches;
    f->macs += real_macs_per_px * (int64_t)B * H * W;
    if (e != cudaSuccess) {
      set_error(std::string("film: streamconv launch failed: ") + cudaGetErrorString(e) + " / " + vfi_last_error());
      return VFI_E_CUDA;
    }
    return VFI_OK;
  }
  int ck(cudaError_t e, const char* what) {
    ++launches;
    if (e != cudaSuccess) {
      set_error(std::string("film: ") + what + ": " + cudaGetErrorString(e));
      return VFI_E_CUDA;
    }
    return VFI_OK;
  }
};

#define RUN(expr)            \
  do {                       \
    const int _rc = (expr);  \
    if (_rc) return _rc;     \
  } while (0)

uint8_t* bp(const Buf& b) { return static_cast<uint8_t*>(b.p); }

// 16-bit element pointer: image `img` of a [n, H_l, W_l, pitch] tensor, channel `ch`
void* at16(const Buf& b, size_t img, size_t px, int pitch, int ch) { return bp(b) + ((img * px) * pitch + ch) * 2; }

int forward(vfi_ctx* c, FilmState* f, const float* frames, int n_frames, int H, int W, int C, const int32_t* f0,
            const int32_t* f1, int B, int clamp01, float* out, cudaStream_t st) {
  if (H < 64 || W < 64) return ffail(VFI_E_INVALID, "film: frames must be at least 64 x 64 (7 pyramid levels)");
  Dims d;
  d.H[0] = H;
  d.W[0] = W;
  for (int l = 1; l < kLevels; ++l) {
    d.H[l] = d.H[l - 1] >> 1;
    d.W[l] = d.W[l - 1] >> 1;
  }
  RUN(ensure_workspace(f, d, B));
  f->last_B = B;
  std::copy(d.H, d.H + kLevels, f->last_H);
  std::copy(d.W, d.W + kLevels, f->last_W);
  Runner r{c, f, ctx_info(c), st};
  const int op = f->op_type;
  f->macs = 0;

  // ---- image pyramids (film_arch.py:395-399, :655-674)
  FilmFrameIdx hidx{};
  for (int i = 0; i < B; ++i) {
    if (f0[i] < 0 || f0[i] >= n_frames || f1[i] < 0 || f1[i] >= n_frames) return ffail(VFI_E_INVALID, "film: frame index");
    hidx.i[i] = f0[i];
    hidx.i[B + i] = f1[i];
  }
  RUN(r.ck(launch_film_gather_rgb(frames, C, hidx, 2 * B, H, W, (float*)f->img[0].p, st), "gather_rgb"));
  for (int l = 1; l < kLevels; ++l)
    RUN(r.ck(launch_film_pool_rgb((const float*)f->img[l - 1].p, (float*)f->img[l].p, 2 * B, d.H[l - 1], d.W[l - 1], st),
             "pool_rgb"));

  // ---- cascaded feature pyramids of both frames (FeatureExtractor.forward :133-163; SubTreeExtractor.forward :102-121)
  for (int i = 0; i < kLevels; ++i) {
    const int n = std::min(kLevels - i, kSub);  // capped sub-levels; deeper ones are never read (:145-146, :158-162)
    for (int j = 0; j < n; ++j) {
      const int l = i + j, cj = 64 << j;
      if (j == 0) {
        RUN(r.ck(launch_film_conv_rgb(op, (const float*)f->img[i].p, f->rgb_w, f->rgb_b, f->tmpA.p, 64, 2 * B, d.H[i], d.W[i], st),
                 "conv_rgb"));
      } else {
        // pool the previous sub-level's output (slice j-1 of feat[l-1]) and run the first conv of this sub-level
        RUN(r.ck(launch_film_pool16(op, at16(f->feat[l - 1], 0, 0, kFeatC[l - 1], kSliceOff[j - 1]), kFeatC[l - 1], f->tmpB.p,
                                    cj / 2, cj / 2, 2 * B, d.H[l - 1], d.W[l - 1], st),
                 "pool16"));
        RUN(r.conv(f->ext[j][0], f->tmpB.p, cj / 2, nullptr, 0, f->tmpA.p, cj, 2 * B, d.H[l], d.W[l], 9ll * (cj / 2) * cj));
      }
      RUN(r.conv(f->ext[j][1], f->tmpA.p, cj, nullptr, 0, at16(f->feat[l], 0, 0, kFeatC[l], kSliceOff[j]), kFeatC[l], 2 * B,
                 d.H[l], d.W[l], 9ll * cj * cj));
    }
  }

  // ---- residual flow pyramids, both directions (PyramidFlowEstimator.forward :567-616); v[dir][l] is the flow of level l
  for (int dir = 0; dir < 2; ++dir) {
    const int a = dir, b = 1 - dir;  // dir 0: forward (frame 0 -> 1), dir 1: backward
    for (int l = kLevels - 1; l >= 0; --l) {
      const int pr = l >= 3 ? 3 : l;
      const int nf = kFlowNF[pr], nfp = std::max(nf, 64), Cl = kFeatC[l];
      const void* fa = at16(f->feat[l], (size_t)a * B, d.px(l), Cl, 0);
      const void* fb = at16(f->feat[l], (size_t)b * B, d.px(l), Cl, 0);
      const float* vup = nullptr;
      if (l < kLevels - 1) {
        RUN(r.ck(launch_film_flow_up((const float*)f->v[dir][l + 1].p, d.H[l + 1], d.W[l + 1], (float*)f->vup.p, B, d.H[l],
                                     d.W[l], st),
                 "flow_up"));
        RUN(r.ck(launch_film_warp16(op, fb, Cl, Cl, (const float*)f->vup.p, 1.f, f->wb.p, Cl, B, d.H[l], d.W[l], st), "warp16"));
        fb = f->wb.p;
        vup = (const float*)f->vup.p;
      }
      RUN(r.conv(f->flow[pr][0], fa, Cl, fb, Cl, f->t0.p, nfp, B, d.H[l], d.W[l], 9ll * 2 * Cl * nf));
      RUN(r.conv(f->flow[pr][1], f->t0.p, nfp, nullptr, 0, f->t1.p, nfp, B, d.H[l], d.W[l], 9ll * nf * nf));
      RUN(r.conv(f->flow[pr][2], f->t1.p, nfp, nullptr, 0, f->t0.p, nfp, B, d.H[l], d.W[l], 9ll * nf * nf));
      RUN(r.conv(f->flow[pr][3], f->t0.p, nfp, nullptr, 0, f->t3.p, nf / 2, B, d.H[l], d.W[l], 1ll * nf * (nf / 2)));
      RUN(r.ck(launch_film_flow_head(op, f->t3.p, nf / 2, nf / 2, f->head_w[pr], f->head_b[pr], vup, (float*)f->v[dir][l].p, B,
                                     d.H[l], d.W[l], st),
               "flow_head"));
    }
  }

  // ---- aligned pyramid (debug_forward :425-447): image 0 is read through the backward flow, image 1 through the forward
  for (int l = 0; l < kFuseLevels; ++l) {
    const int Cl = kFeatC[l], pitch = 2 * Cl + 64;
    const float* bwd = (const float*)f->v[1][l].p;
    const float* fwd = (const float*)f->v[0][l].p;
    RUN(r.ck(launch_film_warp16(op, at16(f->feat[l], 0, d.px(l), Cl, 0), Cl, Cl, bwd, 0.5f, at16(f->aligned[l], 0, 0, pitch, 0),
                                pitch, B, d.H[l], d.W[l], st),
             "warp16"));
    RUN(r.ck(launch_film_warp16(op, at16(f->feat[l], (size_t)B, d.px(l), Cl, 0), Cl, Cl, fwd, 0.5f,
                                at16(f->aligned[l], 0, 0, pitch, Cl), pitch, B, d.H[l], d.W[l], st),
             "warp16"));
    const float* i0 = (const float*)f->img[l].p;
    RUN(r.ck(launch_film_misc64(op, i0, i0 + (size_t)B * d.px(l) * 3, bwd, fwd, at16(f->aligned[l], 0, 0, pitch, 2 * Cl), pitch,
                                B, d.H[l], d.W[l], st),
             "misc64"));
  }

  // ---- fusion (Fusion.forward :258-296)
  const void* net = f->aligned[4].p;
  int net_c = 2 * 960 + 64, net_l = 4;
  const int net_real[4] = {1930, 512, 256, 128};
  for (int k = 0; k < 4; ++k) {
    const int i = 3 - k, nf = (i < 3) ? (64 << i) : 512;
    const int Ca = 2 * kFeatC[i] + 64, Ca_real = 2 * kFeatC[i] + 10;
    RUN(r.ck(launch_film_nearest16(net, d.H[net_l], d.W[net_l], f->upbuf.p, net_c, B, d.H[i], d.W[i], st), "nearest16"));
    RUN(r.conv(f->fuse[k][0], f->upbuf.p, net_c, nullptr, 0, f->n0.p, nf, B, d.H[i], d.W[i], 4ll * net_real[k] * nf));
    RUN(r.conv(f->fuse[k][1], f->aligned[i].p, Ca, f->n0.p, nf, f->n1.p, nf, B, d.H[i], d.W[i], 9ll * (Ca_real + nf) * nf));
    RUN(r.conv(f->fuse[k][2], f->n1.p, nf, nullptr, 0, f->n2.p, nf, B, d.H[i], d.W[i], 9ll * nf * nf));
    net = f->n2.p;
    net_c = nf;
    net_l = i;
  }
  RUN(r.ck(launch_film_out_rgb(op, f->n2.p, 64, f->out_w, f->out_b, clamp01, out, B, H, W, st), "out_rgb"));
  ctx_add_launches(c, r.launches);
  return VFI_OK;
}

}  // namespace
}  // namespace vfi

using namespace vfi;

extern "C" {

// state_dict order: oracle/film.py state_dict_spec (== film_arch.Interpolator().state_dict())
int vfi_film_load(vfi_ctx* c, const float* const* T, const int64_t* numel, int n_tensors, int operand_type) {
  if (!c || !T || !numel) return ffail(VFI_E_INVALID, "null argument");
  if (n_tensors != VFI_FILM_NUM_TENSORS) return ffail(VFI_E_INVALID, "film: expected 82 tensors (Interpolator.state_dict())");
  if (operand_type != VFI_OPERAND_F16 && operand_type != VFI_OPERAND_BF16) return ffail(VFI_E_INVALID, "operand type");
  const CtxInfo ci = ctx_info(c);
  FCK(cudaSetDevice(ci.device));
  film_destroy(ctx_film(c));
  FilmState* f = new FilmState();
  ctx_film(c) = f;
  f->op_type = operand_type;
  int t = 0;
  auto want = [&](int64_t n) { return numel[t] == n; };
  void* d = nullptr;
  // ---- extract.extract_sublevels.convs.{j}.{0,1}
  for (int j = 0; j < kSub; ++j) {
    const int cj = 64 << j, cin = j ? cj / 2 : 3;
    if (!want((int64_t)cj * cin * 9) || numel[t + 1] != cj || numel[t + 2] != (int64_t)cj * cj * 9 || numel[t + 3] != cj)
      return ffail(VFI_E_INVALID, "film: extract tensor sizes");
    if (j == 0) {
      RUN(fupload(f, T[t], (size_t)64 * 27, &d));
      f->rgb_w = (float*)d;
      RUN(fupload(f, T[t + 1], 64, &d));
      f->rgb_b = (float*)d;
    } else {
      RUN(build_conv(f, f->ext[j][0], 3, cin, 0, cj, 1, T[t], T[t + 1], cj, cin, identity_map(cin, cin)));
    }
    RUN(build_conv(f, f->ext[j][1], 3, cj, 0, cj, 1, T[t + 2], T[t + 3], cj, cj, identity_map(cj, cj)));
    t += 4;
  }
  // ---- predict_flow._predictor (shared, levels 3..6), then _predictors.{0,1,2} = levels 2, 1, 0 (film_arch.py:564-565)
  const int order[4] = {3, 2, 1, 0};
  for (int q = 0; q < 4; ++q) {
    const int pr = order[q], nf = kFlowNF[pr], nfp = std::max(nf, 64), Cl = kFeatC[pr];
    const int cin = 2 * Cl;
    if (!want((int64_t)nf * cin * 9) || numel[t + 2] != (int64_t)nf * nf * 9 || numel[t + 4] != (int64_t)nf * nf * 9 ||
        numel[t + 6] != (int64_t)(nf / 2) * nf || numel[t + 8] != (int64_t)2 * (nf / 2) || numel[t + 9] != 2)
      return ffail(VFI_E_INVALID, "film: flow estimator tensor sizes");
    RUN(build_conv(f, f->flow[pr][0], 3, Cl, Cl, nfp, 1, T[t], T[t + 1], nf, cin, identity_map(cin, cin)));
    RUN(build_conv(f, f->flow[pr][1], 3, nfp, 0, nfp, 1, T[t + 2], T[t + 3], nf, nf, identity_map(nf, nfp)));
    RUN(build_conv(f, f->flow[pr][2], 3, nfp, 0, nfp, 1, T[t + 4], T[t + 5], nf, nf, identity_map(nf, nfp)));
    RUN(build_conv(f, f->flow[pr][3], 1, nfp, 0, nf / 2, 1, T[t + 6], T[t + 7], nf / 2, nf, identity_map(nf, nfp)));
    RUN(fupload(f, T[t + 8], (size_t)2 * (nf / 2), &d));
    f->head_w[pr] = (float*)d;
    RUN(fupload(f, T[t + 9], 2, &d));
    f->head_b[pr] = (float*)d;
    t += 10;
  }
  // ---- fuse.output_conv, fuse.convs.{k}.{0,1,2} (film_arch.py:230, :243-256)
  if (!want(3 * 64) || numel[t + 1] != 3) return ffail(VFI_E_INVALID, "film: output conv sizes");
  RUN(fupload(f, T[t], 3 * 64, &d));
  f->out_w = (float*)d;
  RUN(fupload(f, T[t + 1], 3, &d));
  f->out_b = (float*)d;
  t += 2;
  int net_real = 2 * 960 + 10, net_pad = 2 * 960 + 64;
  std::vector<int> net_map = aligned_map(960);
  for (int k = 0; k < 4; ++k) {
    const int i = 3 - k, nf = (i < 3) ? (64 << i) : 512;
    const int Ca = 2 * kFeatC[i] + 64, Ca_real = 2 * kFeatC[i] + 10;
    if (!want((int64_t)nf * net_real * 4) || numel[t + 2] != (int64_t)nf * (Ca_real + nf) * 9 ||
        numel[t + 4] != (int64_t)nf * nf * 9)
      return ffail(VFI_E_INVALID, "film: fusion tensor sizes");
    RUN(build_conv(f, f->fuse[k][0], 2, net_pad, 0, nf, 0, T[t], T[t + 1], nf, net_real, net_map));
    std::vector<int> m = aligned_map(kFeatC[i]);
    for (int j = 0; j < nf; ++j) m.push_back(Ca_real + j);
    RUN(build_conv(f, f->fuse[k][1], 3, Ca, nf, nf, 1, T[t + 2], T[t + 3], nf, Ca_real + nf, m));
    RUN(build_conv(f, f->fuse[k][2], 3, nf, 0, nf, 1, T[t + 4], T[t + 5], nf, nf, identity_map(nf, nf)));
    t += 6;
    net_real = nf;
    net_pad = nf;
    net_map = identity_map(nf, nf);
  }
  if (t != VFI_FILM_NUM_TENSORS) return ffail(VFI_E_INVALID, "film: internal tensor count");
  f->loaded = true;
  return VFI_OK;
}

int vfi_film_forward(vfi_ctx* c, const float* frames, int n_frames, int H, int W, int C, const int32_t* f0,
                     const int32_t* f1, int n_pairs, int clamp01, float* out, void* stream) {
  if (!c || !frames || !f0 || !f1 || !out) return ffail(VFI_E_INVALID, "null argument");
  FilmState* f = ctx_film(c);
  if (!f || !f->loaded) return ffail(VFI_E_STATE, "vfi_film_load has not been called");
  if (n_pairs < 1 || n_pairs > kMaxBatch) return ffail(VFI_E_INVALID, "film: n_pairs must be in [1,16]");
  if (C < 3) return ffail(VFI_E_INVALID, "film: frames need >= 3 channels");
  FCK(cudaSetDevice(ctx_info(c).device));
  return forward(c, f, frames, n_frames, H, W, C, f0, f1, n_pairs, clamp01, out, static_cast<cudaStream_t>(stream));
}

int vfi_film_debug_set_ref(vfi_ctx* c, int use_ref) {
  FilmState* f = c ? ctx_film(c) : nullptr;
  if (!f) return ffail(VFI_E_STATE, "vfi_film_load has not been called");
  f->use_ref = use_ref != 0;
  return VFI_OK;
}

/* group 0 = extract (layer = 2*j + which, j >= 1 or which = 1), 1 = flow (layer = 4*predictor + conv), 2 = fuse (3*k + conv) */
int vfi_film_debug_conv(vfi_ctx* c, int group, int layer, const void* src0, int pitch0, const void* src1, int pitch1,
                        void* out, int out_pitch, int B, int H, int W, int impl, void* stream) {
  FilmState* f = c ? ctx_film(c) : nullptr;
  if (!f || !f->loaded) return ffail(VFI_E_STATE, "vfi_film_load has not been called");
  const StreamConvLayer* L = nullptr;
  if (group == 0 && layer >= 1 && layer < 8 && layer != 0) L = &f->ext[layer / 2][layer % 2];
  if (group == 1 && layer >= 0 && layer < 16) L = &f->flow[layer / 4][layer % 4];
  if (group == 2 && layer >= 0 && layer < 12) L = &f->fuse[layer / 3][layer % 3];
  if (!L || !L->w) return ffail(VFI_E_INVALID, "film: no such conv layer");
  FCK(cudaSetDevice(ctx_info(c).device));
  const cudaError_t e = launch_streamconv(*L, f->op_type, src0, pitch0, src1, pitch1, out, out_pitch, B, H, W,
                                          ctx_info(c).num_sms, impl != 0, static_cast<cudaStream_t>(stream));
  ctx_add_launches(c, 1);
  if (e != cudaSuccess) return ffail(VFI_E_CUDA, std::string("streamconv: ") + cudaGetErrorString(e) + " / " + vfi_last_error());
  return VFI_OK;
}

int vfi_film_debug_state(vfi_ctx* c, int dir, int level, float* out, int batch, int* H, int* W) {
  FilmState* f = c ? ctx_film(c) : nullptr;
  if (!f || !f->loaded) return ffail(VFI_E_STATE, "vfi_film_load has not been called");
  if (!H || !W) return ffail(VFI_E_INVALID, "null argument");
  if (dir < 0 || dir > 1 || level < 0 || level >= kLevels) return ffail(VFI_E_INVALID, "film: no such flow level");
  if (!f->last_B) return ffail(VFI_E_STATE, "film: no forward has run");
  FCK(cudaSetDevice(ctx_info(c).device));
  FCK(cudaDeviceSynchronize());
  *H = f->last_H[level];
  *W = f->last_W[level];
  if (!out) return VFI_OK;
  if (batch < 1 || batch > f->last_B) return ffail(VFI_E_INVALID, "film: batch larger than the last forward");
  FCK(cudaMemcpy(out, f->v[dir][level].p, (size_t)batch * *H * *W * 2 * sizeof(float), cudaMemcpyDeviceToDevice));
  FCK(cudaDeviceSynchronize());
  return VFI_OK;
}

int vfi_film_debug_elem(vfi_ctx* c, int kernel, const void* in0, int in_pitch, const void* in1, const void* in2,
                        const void* in3, const int32_t* frame_idx, void* out, int out_pitch, int C, int B, int H, int W,
                        int h, int w, float fscale, int clamp01, int predictor, void* stream) {
  FilmState* f = c ? ctx_film(c) : nullptr;
  if (!f || !f->loaded) return ffail(VFI_E_STATE, "vfi_film_load has not been called");
  if (B < 1 || H < 1 || W < 1) return ffail(VFI_E_INVALID, "film: empty launch");
  const int op = f->op_type;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  FCK(cudaSetDevice(ctx_info(c).device));
  cudaError_t e = cudaSuccess;
  switch (kernel) {
    case 0: {
      if (B > 2 * kMaxBatch || !frame_idx) return ffail(VFI_E_INVALID, "film: gather_rgb takes 1..32 frame indices");
      FilmFrameIdx idx{};
      for (int i = 0; i < B; ++i) idx.i[i] = frame_idx[i];
      e = launch_film_gather_rgb((const float*)in0, C, idx, B, H, W, (float*)out, st);
      break;
    }
    case 1: e = launch_film_pool_rgb((const float*)in0, (float*)out, B, H, W, st); break;
    case 2: e = launch_film_conv_rgb(op, (const float*)in0, f->rgb_w, f->rgb_b, out, out_pitch, B, H, W, st); break;
    case 3: e = launch_film_pool16(op, in0, in_pitch, out, out_pitch, C, B, H, W, st); break;
    case 4: e = launch_film_flow_up((const float*)in0, h, w, (float*)out, B, H, W, st); break;
    case 5: e = launch_film_warp16(op, in0, in_pitch, C, (const float*)in1, fscale, out, out_pitch, B, H, W, st); break;
    case 6:
      e = launch_film_misc64(op, (const float*)in0, (const float*)in1, (const float*)in2, (const float*)in3, out, out_pitch,
                             B, H, W, st);
      break;
    case 7: e = launch_film_nearest16(in0, h, w, out, C, B, H, W, st); break;
    case 8:
      if (predictor < 0 || predictor > 3) return ffail(VFI_E_INVALID, "film: no such flow predictor");
      if (C <= 128 && C != kFlowNF[predictor] / 2)
        return ffail(VFI_E_INVALID, "film: flow_head of predictor " + std::to_string(predictor) + " reads " +
                                        std::to_string(kFlowNF[predictor] / 2) + " channels");
      e = launch_film_flow_head(op, in0, in_pitch, C, f->head_w[predictor], f->head_b[predictor], (const float*)in1,
                                (float*)out, B, H, W, st);
      break;
    case 9: e = launch_film_out_rgb(op, in0, in_pitch, f->out_w, f->out_b, clamp01, (float*)out, B, H, W, st); break;
    default: return ffail(VFI_E_INVALID, "film: no such element-wise kernel");
  }
  ctx_add_launches(c, 1);
  if (e == cudaErrorInvalidValue) {  // the launchers' refusals, named
    if ((kernel == 3 || kernel == 5 || kernel == 7 || kernel == 8) && (C & 7))
      return ffail(VFI_E_INVALID, "film: C must be a multiple of 8");
    if (kernel == 8) return ffail(VFI_E_INVALID, "film: flow_head reads at most 128 channels");
    if (kernel == 1 || kernel == 3) return ffail(VFI_E_INVALID, "film: level too small to pool");
    return ffail(VFI_E_INVALID, "film: launch refused");
  }
  if (e != cudaSuccess) return ffail(VFI_E_CUDA, std::string("film: element-wise launch: ") + cudaGetErrorString(e));
  return VFI_OK;
}

int vfi_film_layer_plan(vfi_ctx* c, int group, int layer, int* c0, int* c1, int* n_total, int* ksize, int* n_cta,
                        int* nsplit, int* mt, int* a_slots, int* b_slots, int* smem_bytes) {
  FilmState* f = c ? ctx_film(c) : nullptr;
  if (!f || !f->loaded) return ffail(VFI_E_STATE, "vfi_film_load has not been called");
  const StreamConvLayer* L = nullptr;
  if (group == 0 && layer >= 1 && layer < 8) L = &f->ext[layer / 2][layer % 2];
  if (group == 1 && layer >= 0 && layer < 16) L = &f->flow[layer / 4][layer % 4];
  if (group == 2 && layer >= 0 && layer < 12) L = &f->fuse[layer / 3][layer % 3];
  if (!L || !L->w) return ffail(VFI_E_INVALID, "film: no such conv layer");
  StreamConvParams p{};
  if (!streamconv_plan(*L, &p)) return ffail(VFI_E_INVALID, "film: plan failed");
  if (c0) *c0 = L->c0;
  if (c1) *c1 = L->c1;
  if (n_total) *n_total = L->n_total;
  if (ksize) *ksize = L->ksize;
  if (n_cta) *n_cta = p.n_cta;
  if (nsplit) *nsplit = p.nsplit;
  if (mt) *mt = p.mt;
  if (a_slots) *a_slots = p.a_slots;
  if (b_slots) *b_slots = p.b_slots;
  if (smem_bytes) *smem_bytes = (int)p.smem_bytes;
  return VFI_OK;
}

/* Host-only (no GPU needed): the weight packer and channel maps of vfi_film_load on caller data.  layout 0: input
 * channels in reference order, `cin` real of c0 = ceil64(cin) padded; layout 1: the fusion input of a level with C
 * feature channels per frame, [wfeat0 C | wfeat1 C | misc 64] (+ nf channels of the decoder state in a second tensor). */
int vfi_film_debug_pack_host(int layout, int C, int nf, int ksize, int n_total, int operand_type, const float* w,
                             int cout, int cin, uint16_t* out, int64_t out_cap, int* c0, int* c1, int* n_cta,
                             int* nsplit) {
  if (!w || !out) return ffail(VFI_E_INVALID, "null argument");
  std::vector<int> m;
  int k0 = 0, k1 = 0;
  if (layout == 0) {
    k0 = (cin + 63) / 64 * 64;
    m = identity_map(cin, k0);
  } else if (layout == 1) {
    m = aligned_map(C);
    k0 = 2 * C + 64;
    k1 = nf;
    for (int j = 0; j < nf; ++j) m.push_back(2 * C + 10 + j);
  } else {
    return ffail(VFI_E_INVALID, "layout");
  }
  std::vector<uint16_t> pk;
  StreamConvParams p{};
  const int rc = pack_conv(operand_type, ksize, k0, k1, n_total, w, cout, cin, m, &pk, &p);
  if (rc) return rc;
  if ((int64_t)pk.size() > out_cap) return ffail(VFI_E_INVALID, "output buffer too small");
  std::memcpy(out, pk.data(), pk.size() * 2);
  if (c0) *c0 = k0;
  if (c1) *c1 = k1;
  if (n_cta) *n_cta = p.n_cta;
  if (nsplit) *nsplit = p.nsplit;
  return VFI_OK;
}

int64_t vfi_film_last_macs(const vfi_ctx* c) {
  FilmState* f = c ? ctx_film(const_cast<vfi_ctx*>(c)) : nullptr;
  return f ? f->macs : 0;
}

}  // extern "C"
