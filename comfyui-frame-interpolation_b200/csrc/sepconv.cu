// Sepconv ("revisiting adaptive convolutions", the reference's `Sepconv VFI` node) on H100: weights, workspace, forward
// schedule and C ABI.  SURVEY.md section 8 row a12.  Reference: vfi_models/sepconv/sepconv_enhanced.py, Network :536-706.
//
// Forward for B pairs (levels: row 0 = He x We (input padded to even), row r = ceil(row r-1 / 2); C_r = 32,64,128,256,512):
//   sep_stats, sep_input_conv         normalise the pair, netInput on both frames, cat, PReLU, space-to-depth   :620-642
//   rows 1..4 (Encode.netVer)         [prelu_s2d16 ->] streamconv 2x2 over the space-to-depth grid (= the 3x3 stride-2
//                                     conv, padding row/column before) + PReLU -> streamconv 3x3                  :549-556
//   rows 4..1 (Decode.netHor)         prelu16 -> streamconv 3x3 + PReLU -> streamconv 3x3 + skip (in place)       :571-576
//   rows 3..1 (Decode.netVer)         prelu_up2_16 (PReLU, bilinear x2, crop) -> streamconv + PReLU -> streamconv
//                                     added onto the row (in place)                                                :577-580, :479-496
//   4 heads                           prelu_up2_16 (no PReLU) once; per head streamconv + PReLU -> streamconv to 51
//                                     (padded 64) columns -> sep_coeff_nchw                                        :583-598, :683-686
//   sep_pad_input x2, sepconv op x2   the adaptive separable convolution (ops.cu, the kernel behind vfi_sepconv)    :644-690
//   sep_finish                        normalise by the ones channel, crop, NHWC                                    :692-702
// All convs run on streamconv.cu's EXT epilogue (learned PReLU slope, residual).  The first version keeps the verified op
// kernel's NCHW fp32 interface (coefficients transposed by sep_coeff_nchw); fusing that transpose into the op is the
// obvious next step once this path has been timed.
#include <cuda_fp16.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <cstring>
#include <string>

#include "../../include/vfi_b200.h"
#include "vfi_internal.h"

namespace vfi {

namespace {
constexpr int kRows = 5, kK = 51;
const int kC[kRows] = {32, 64, 128, 256, 512};

struct SBuf {
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

struct SepState {
  int op_type = OP_F16;
  bool loaded = false;
  bool use_ref = false;
  std::vector<void*> allocs;
  float* in_w = nullptr;  // netInput (CUDA cores)
  float* in_b = nullptr;
  float enc_s0[kRows] = {0}, dec_s0[kRows] = {0}, up_s0[kRows] = {0};  // PReLU applied by the element-wise pre-pass of a row
  StreamConvLayer enc[kRows][2];  // [row 1..4][stride-2 conv as 2x2 over s2d, 3x3]
  StreamConvLayer hor[kRows][2];  // [row 1..4][3x3 + PReLU, 3x3 + skip]
  StreamConvLayer ver[kRows][2];  // [row 1..3][3x3 C_{r+1} -> C_r + PReLU, 3x3 added onto the row]
  StreamConvLayer head[4][2];     // Verone, Vertwo, Horone, Hortwo: [3x3 64 -> 64 + PReLU, 3x3 64 -> 51 (64 columns)]
  SBuf x[kRows], S, T, U, V, K, coef[4], P1, P2, O1, O2, stats, statp;
  int last_B = 0;  // pairs and row sizes of the last forward (vfi_sepconv_debug_state)
  int last_h[kRows] = {}, last_w[kRows] = {};
};

void sepconv_destroy(SepState* s) {
  if (!s) return;
  for (void* p : s->allocs) cudaFree(p);
  for (int r = 0; r < kRows; ++r) s->x[r].release();
  for (SBuf* b : {&s->S, &s->T, &s->U, &s->V, &s->K, &s->coef[0], &s->coef[1], &s->coef[2], &s->coef[3], &s->P1, &s->P2, &s->O1,
                  &s->O2, &s->stats, &s->statp})
    b->release();
  delete s;
}

namespace {

#define SCK(call)                                                            \
  do {                                                                       \
    cudaError_t _e = (call);                                                 \
    if (_e != cudaSuccess) {                                                 \
      set_error(std::string(#call) + ": " + cudaGetErrorString(_e));         \
      return VFI_E_CUDA;                                                     \
    }                                                                        \
  } while (0)
#define SRUN(expr)           \
  do {                       \
    const int _rc = (expr);  \
    if (_rc) return _rc;     \
  } while (0)

int sfail(int code, const std::string& msg) {
  set_error(msg);
  return code;
}

template <class T>
int supload(SepState* s, const T* h, size_t n, void** dptr) {
  void* d = nullptr;
  SCK(cudaMalloc(&d, n * sizeof(T)));
  s->allocs.push_back(d);
  SCK(cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice));
  *dptr = d;
  return VFI_OK;
}

// A 3x3 stride-1 conv [cout][cin][3][3] (pad 1), cin a multiple of 64; `slope` = PReLU after it (1 = none).
// stride2 = true: the same weights as a 2x2 conv over the space-to-depth input [(a, b, cin)] with one padding row / column
// BEFORE: tap (ty, tx) at cell offset (ty - 1, tx - 1) and sub-pixel (a, b) is kernel element (2 ty + a - 1, 2 tx + b - 1).
int build(SepState* s, StreamConvLayer& L, bool stride2, int cin, int cout, int n_total, float slope, const float* w,
          const float* bias) {
  L = StreamConvLayer{};
  L.ext = 1;
  L.slope = slope;
  L.act = 0;
  L.n_total = n_total;
  L.c1 = 0;
  if (stride2) {
    L.ksize = 2;
    L.pad_before = 1;
    L.c0 = 4 * cin;
  } else {
    L.ksize = 3;
    L.c0 = cin;
  }
  std::vector<uint16_t> pk;
  StreamConvParams p{};
  const bool ok = pack_streamconv(L, s->op_type, [&](int n, int tap, int j) -> float {
    if (n >= cout) return 0.f;
    if (!stride2) return w[((size_t)n * cin + j) * 9 + tap];
    const int ab = j / cin, c = j - ab * cin;
    const int ky = 2 * (tap >> 1) + (ab >> 1) - 1, kx = 2 * (tap & 1) + (ab & 1) - 1;
    if (ky < 0 || kx < 0) return 0.f;  // (ky, kx <= 2 always)
    return w[((size_t)n * cin + c) * 9 + ky * 3 + kx];
  }, &pk, &p);
  if (!ok) return sfail(VFI_E_INVALID, "sepconv: layer shape not supported by streamconv");
  std::vector<float> sh(n_total, 0.f);
  for (int n = 0; n < cout; ++n) sh[n] = bias[n];
  SRUN(supload(s, pk.data(), pk.size(), &L.w));
  void* d = nullptr;
  SRUN(supload(s, sh.data(), sh.size(), &d));
  L.shift = static_cast<float*>(d);
  return VFI_OK;
}

struct SRunner {
  vfi_ctx* c;
  SepState* s;
  int num_sms;
  cudaStream_t st;
  int launches = 0;
  int conv(const StreamConvLayer& L, const void* in, void* out, int B, int H, int W, const void* res = nullptr) {
    const cudaError_t e = launch_streamconv(L, s->op_type, in, L.c0, nullptr, 0, out, L.n_total, B, H, W, num_sms, s->use_ref,
                                            st, res);
    ++launches;
    if (e != cudaSuccess) {
      set_error(std::string("sepconv: streamconv launch failed: ") + cudaGetErrorString(e) + " / " + vfi_last_error());
      return VFI_E_CUDA;
    }
    return VFI_OK;
  }
  int ck(cudaError_t e, const char* what) {
    ++launches;
    if (e != cudaSuccess) {
      set_error(std::string("sepconv: ") + what + ": " + cudaGetErrorString(e));
      return VFI_E_CUDA;
    }
    return VFI_OK;
  }
};

int forward(vfi_ctx* c, SepState* s, const float* frames, int n_frames, int H, int W, int C, const int32_t* f0,
            const int32_t* f1, int B, float* out, cudaStream_t st) {
  const int He = H + (H & 1), We = W + (W & 1);
  int h[kRows], w[kRows];
  h[0] = He;
  w[0] = We;
  for (int r = 1; r < kRows; ++r) {
    h[r] = (h[r - 1] + 1) / 2;
    w[r] = (w[r - 1] + 1) / 2;
  }
  SepPairIdx idx{};
  for (int i = 0; i < B; ++i) {
    if (f0[i] < 0 || f0[i] >= n_frames || f1[i] < 0 || f1[i] >= n_frames) return sfail(VFI_E_INVALID, "sepconv: frame index");
    idx.f0[i] = f0[i];
    idx.f1[i] = f1[i];
  }
  const size_t px0 = (size_t)He * We;
  for (int r = 1; r < kRows; ++r) SCK(s->x[r].ensure((size_t)B * h[r] * w[r] * kC[r] * 2));
  size_t nS = 0, nT = px0 * 64, nU = px0 * 64;  // elements per pair: s2d inputs, conv scratch, activated / up-sampled inputs
  for (int r = 1; r < kRows; ++r) {
    nS = std::max(nS, (size_t)h[r] * w[r] * 4 * kC[r - 1]);
    nT = std::max(nT, (size_t)h[r] * w[r] * kC[r]);
    nU = std::max(nU, (size_t)h[r] * w[r] * kC[r]);
    if (r < kRows - 1) {  // Decode.netVer runs at the up-sampled size 2 h[r+1] x 2 w[r+1] and is cropped when added
      nT = std::max(nT, (size_t)4 * h[r + 1] * w[r + 1] * kC[r]);
      nU = std::max(nU, (size_t)4 * h[r + 1] * w[r + 1] * kC[r + 1]);
    }
  }
  SCK(s->S.ensure((size_t)B * nS * 2));
  SCK(s->T.ensure((size_t)B * nT * 2));
  SCK(s->U.ensure((size_t)B * nU * 2));
  SCK(s->V.ensure((size_t)B * nT * 2));
  SCK(s->K.ensure((size_t)B * px0 * 64 * 2));
  for (int k = 0; k < 4; ++k) SCK(s->coef[k].ensure((size_t)B * kK * px0 * 4));
  const int Hp = He + kK - 1, Wp = We + kK - 1;
  SCK(s->P1.ensure((size_t)B * 4 * Hp * Wp * 4));
  SCK(s->P2.ensure((size_t)B * 4 * Hp * Wp * 4));
  SCK(s->O1.ensure((size_t)B * 4 * px0 * 4));
  SCK(s->O2.ensure((size_t)B * 4 * px0 * 4));
  SCK(s->stats.ensure(2 * kMaxBatch * sizeof(double)));
  SCK(s->statp.ensure((size_t)B * sep_stats_blocks(He, We) * 2 * sizeof(double)));
  s->last_B = B;
  std::copy(h, h + kRows, s->last_h);
  std::copy(w, w + kRows, s->last_w);
  SRunner r{c, s, ctx_info(c).num_sms, st};
  const int op = s->op_type;

  SRUN(r.ck(launch_sep_stats(frames, C, idx, B, H, W, He, We, (double*)s->stats.p, (double*)s->statp.p, st), "sep_stats"));
  SRUN(r.ck(launch_sep_input_conv(op, frames, C, idx, B, H, W, He, We, (const double*)s->stats.p, s->in_w, s->in_b,
                                  s->enc_s0[1], s->S.p, st),
            "sep_input_conv"));
  // ---- Encode: rows 1..4
  for (int row = 1; row < kRows; ++row) {
    if (row > 1)
      SRUN(r.ck(launch_prelu_s2d16(op, s->x[row - 1].p, s->S.p, s->enc_s0[row], kC[row - 1], B, h[row - 1], w[row - 1], st),
                "prelu_s2d16"));
    SRUN(r.conv(s->enc[row][0], s->S.p, s->T.p, B, h[row], w[row]));
    SRUN(r.conv(s->enc[row][1], s->T.p, s->x[row].p, B, h[row], w[row]));
  }
  // ---- Decode: Hor on rows 4..1 (in place: x += conv(prelu(conv(prelu(x)))))
  for (int row = kRows - 1; row >= 1; --row) {
    SRUN(r.ck(launch_prelu16(op, s->x[row].p, s->U.p, s->dec_s0[row], (size_t)B * h[row] * w[row] * kC[row], st), "prelu16"));
    SRUN(r.conv(s->hor[row][0], s->U.p, s->T.p, B, h[row], w[row]));
    SRUN(r.conv(s->hor[row][1], s->T.p, s->x[row].p, B, h[row], w[row], s->x[row].p));
  }
  // ---- Decode: Ver on rows 3..1: x_r += conv(prelu(conv(up(prelu(x_{r+1}))))).  The reference runs both convs at the
  // up-sampled size and THEN crops a surplus row / column (:479-494), so with an odd row size the convs see real data
  // where a crop-first order would see zero padding: run them at 2 h[r+1] x 2 w[r+1] and crop in the add.
  for (int row = kRows - 2; row >= 1; --row) {
    const int hu = 2 * h[row + 1], wu = 2 * w[row + 1];
    SRUN(r.ck(launch_prelu_up2_16(op, s->x[row + 1].p, s->U.p, s->up_s0[row], kC[row + 1], B, h[row + 1], w[row + 1], hu, wu, st),
              "prelu_up2_16"));
    SRUN(r.conv(s->ver[row][0], s->U.p, s->T.p, B, hu, wu));
    if (hu == h[row] && wu == w[row]) {
      SRUN(r.conv(s->ver[row][1], s->T.p, s->x[row].p, B, hu, wu, s->x[row].p));
    } else {
      SRUN(r.conv(s->ver[row][1], s->T.p, s->V.p, B, hu, wu));
      SRUN(r.ck(launch_add_crop16(op, s->V.p, hu, wu, s->x[row].p, kC[row], B, h[row], w[row], st), "add_crop16"));
    }
  }
  // ---- heads: up(row 1) once, then conv-prelu-conv per head
  SRUN(r.ck(launch_prelu_up2_16(op, s->x[1].p, s->U.p, 1.f, 64, B, h[1], w[1], He, We, st), "prelu_up2_16"));
  for (int k = 0; k < 4; ++k) {
    SRUN(r.conv(s->head[k][0], s->U.p, s->T.p, B, He, We));
    SRUN(r.conv(s->head[k][1], s->T.p, s->K.p, B, He, We));
    SRUN(r.ck(launch_sep_coeff_nchw(op, s->K.p, 64, (float*)s->coef[k].p, kK, B, He, We, st), "sep_coeff_nchw"));
  }
  // ---- the separable convolution on both frames (heads: 0 Verone, 1 Vertwo, 2 Horone, 3 Hortwo), :688-690
  SRUN(r.ck(launch_sep_pad_input(frames, C, idx, 0, B, H, W, Hp, Wp, (float*)s->P1.p, st), "sep_pad_input"));
  SRUN(r.ck(launch_sep_pad_input(frames, C, idx, 1, B, H, W, Hp, Wp, (float*)s->P2.p, st), "sep_pad_input"));
  SRUN(r.ck(launch_sepconv((const float*)s->P1.p, (const float*)s->coef[0].p, (const float*)s->coef[2].p, (float*)s->O1.p, B, 4,
                           He, We, kK, kK, st),
            "sepconv op"));
  SRUN(r.ck(launch_sepconv((const float*)s->P2.p, (const float*)s->coef[1].p, (const float*)s->coef[3].p, (float*)s->O2.p, B, 4,
                           He, We, kK, kK, st),
            "sepconv op"));
  SRUN(r.ck(launch_sep_finish((const float*)s->O1.p, (const float*)s->O2.p, out, B, H, W, He, We, st), "sep_finish"));
  ctx_add_launches(c, r.launches);
  return VFI_OK;
}

}  // namespace
}  // namespace vfi

using namespace vfi;

extern "C" {

/* state_dict order: oracle/sepconv.py state_dict_spec (== sepconv_enhanced.Network().state_dict()) */
int vfi_sepconv_load(vfi_ctx* c, const float* const* T, const int64_t* numel, int n_tensors, int operand_type) {
  if (!c || !T || !numel) return sfail(VFI_E_INVALID, "null argument");
  if (n_tensors != VFI_SEPCONV_NUM_TENSORS) return sfail(VFI_E_INVALID, "sepconv: expected 88 tensors (Network.state_dict())");
  if (operand_type != VFI_OPERAND_F16 && operand_type != VFI_OPERAND_BF16) return sfail(VFI_E_INVALID, "operand type");
  SCK(cudaSetDevice(ctx_info(c).device));
  sepconv_destroy(ctx_sep(c));
  SepState* s = new SepState();
  ctx_sep(c) = s;
  s->op_type = operand_type;
  auto chk = [&](int t, int64_t n) { return numel[t] == n; };
  void* d = nullptr;
  if (!chk(0, 16 * 27) || !chk(1, 16)) return sfail(VFI_E_INVALID, "sepconv: netInput sizes");
  SRUN(supload(s, T[0], 16 * 27, &d));
  s->in_w = (float*)d;
  SRUN(supload(s, T[1], 16, &d));
  s->in_b = (float*)d;
  int t = 2;
  // Encode.netVer rows 1..4: prelu, sconv, prelu, conv
  for (int r = 1; r < kRows; ++r, t += 6) {
    const int ci = kC[r - 1], co = kC[r];
    if (!chk(t, 1) || !chk(t + 1, (int64_t)co * ci * 9) || !chk(t + 2, co) || !chk(t + 3, 1) ||
        !chk(t + 4, (int64_t)co * co * 9) || !chk(t + 5, co))
      return sfail(VFI_E_INVALID, "sepconv: encoder tensor sizes");
    s->enc_s0[r] = T[t][0];
    SRUN(build(s, s->enc[r][0], true, ci, co, co, T[t + 3][0], T[t + 1], T[t + 2]));
    SRUN(build(s, s->enc[r][1], false, co, co, co, 1.f, T[t + 4], T[t + 5]));
  }
  // Decode.netHor.{0..3} = rows 4, 3, 2, 1: prelu, conv, prelu, conv (+ skip)
  for (int r = kRows - 1; r >= 1; --r, t += 6) {
    const int co = kC[r];
    if (!chk(t, 1) || !chk(t + 1, (int64_t)co * co * 9) || !chk(t + 2, co) || !chk(t + 3, 1) ||
        !chk(t + 4, (int64_t)co * co * 9) || !chk(t + 5, co))
      return sfail(VFI_E_INVALID, "sepconv: decoder (hor) tensor sizes");
    s->dec_s0[r] = T[t][0];
    SRUN(build(s, s->hor[r][0], false, co, co, co, T[t + 3][0], T[t + 1], T[t + 2]));
    SRUN(build(s, s->hor[r][1], false, co, co, co, 1.f, T[t + 4], T[t + 5]));
  }
  // Decode.netVer.{1..3} = rows 3, 2, 1: prelu, up, conv, prelu, conv
  for (int r = kRows - 2; r >= 1; --r, t += 6) {
    const int ci = kC[r + 1], co = kC[r];
    if (!chk(t, 1) || !chk(t + 1, (int64_t)co * ci * 9) || !chk(t + 2, co) || !chk(t + 3, 1) ||
        !chk(t + 4, (int64_t)co * co * 9) || !chk(t + 5, co))
      return sfail(VFI_E_INVALID, "sepconv: decoder (ver) tensor sizes");
    s->up_s0[r] = T[t][0];
    SRUN(build(s, s->ver[r][0], false, ci, co, co, T[t + 3][0], T[t + 1], T[t + 2]));
    SRUN(build(s, s->ver[r][1], false, co, co, co, 1.f, T[t + 4], T[t + 5]));
  }
  // heads Verone, Vertwo, Horone, Hortwo: (up) conv, prelu, conv
  for (int k = 0; k < 4; ++k, t += 5) {
    if (!chk(t, 64 * 64 * 9) || !chk(t + 1, 64) || !chk(t + 2, 1) || !chk(t + 3, (int64_t)kK * 64 * 9) || !chk(t + 4, kK))
      return sfail(VFI_E_INVALID, "sepconv: head tensor sizes");
    SRUN(build(s, s->head[k][0], false, 64, 64, 64, T[t + 2][0], T[t], T[t + 1]));
    SRUN(build(s, s->head[k][1], false, 64, kK, 64, 1.f, T[t + 3], T[t + 4]));
  }
  if (t != VFI_SEPCONV_NUM_TENSORS) return sfail(VFI_E_INVALID, "sepconv: internal tensor count");
  s->loaded = true;
  return VFI_OK;
}

int vfi_sepconv_forward(vfi_ctx* c, const float* frames, int n_frames, int H, int W, int C, const int32_t* f0,
                        const int32_t* f1, int n_pairs, float* out, void* stream) {
  if (!c || !frames || !f0 || !f1 || !out) return sfail(VFI_E_INVALID, "null argument");
  SepState* s = ctx_sep(c);
  if (!s || !s->loaded) return sfail(VFI_E_STATE, "vfi_sepconv_load has not been called");
  if (n_pairs < 1 || n_pairs > kMaxBatch) return sfail(VFI_E_INVALID, "sepconv: n_pairs must be in [1,16]");
  if (C < 3 || H < 2 || W < 2) return sfail(VFI_E_INVALID, "sepconv: frames need >= 3 channels and >= 2 x 2 pixels");
  SCK(cudaSetDevice(ctx_info(c).device));
  return forward(c, s, frames, n_frames, H, W, C, f0, f1, n_pairs, out, static_cast<cudaStream_t>(stream));
}

int vfi_sepconv_debug_set_ref(vfi_ctx* c, int use_ref) {
  SepState* s = c ? ctx_sep(c) : nullptr;
  if (!s) return sfail(VFI_E_STATE, "vfi_sepconv_load has not been called");
  s->use_ref = use_ref != 0;
  return VFI_OK;
}

int vfi_sepconv_debug_state(vfi_ctx* c, int what, int index, void* out, int batch, int* shape) {
  SepState* s = c ? ctx_sep(c) : nullptr;
  if (!s || !s->loaded) return sfail(VFI_E_STATE, "vfi_sepconv_load has not been called");
  if (!shape) return sfail(VFI_E_INVALID, "null argument");
  if (!s->last_B) return sfail(VFI_E_STATE, "sepconv: no forward has run");
  const int He = s->last_h[0], We = s->last_w[0];
  size_t elem = 0;
  const void* src = nullptr;
  if (what == 0) {
    if (index < 0 || index > 3) return sfail(VFI_E_INVALID, "sepconv: no such coefficient plane (0..3)");
    const int sh[4] = {batch, kK, He, We};
    std::copy(sh, sh + 4, shape);
    elem = sizeof(float);
    src = s->coef[index].p;
  } else if (what == 1) {
    if (index < 1 || index >= kRows) return sfail(VFI_E_INVALID, "sepconv: no such pyramid row (1..4)");
    const int sh[4] = {batch, s->last_h[index], s->last_w[index], kC[index]};
    std::copy(sh, sh + 4, shape);
    elem = 2;
    src = s->x[index].p;
  } else if (what == 2) {
    if (index != 0) return sfail(VFI_E_INVALID, "sepconv: the stats have no index");
    const int sh[4] = {batch, 2, 1, 1};
    std::copy(sh, sh + 4, shape);
    elem = sizeof(double);
    src = s->stats.p;
  } else {
    return sfail(VFI_E_INVALID, "sepconv: no such state (0 planes, 1 rows, 2 stats)");
  }
  if (!out) return VFI_OK;
  if (batch < 1 || batch > s->last_B) return sfail(VFI_E_INVALID, "sepconv: batch larger than the last forward");
  SCK(cudaSetDevice(ctx_info(c).device));
  SCK(cudaDeviceSynchronize());
  SCK(cudaMemcpy(out, src, (size_t)shape[0] * shape[1] * shape[2] * shape[3] * elem, cudaMemcpyDeviceToDevice));
  SCK(cudaDeviceSynchronize());
  return VFI_OK;
}

int vfi_sepconv_debug_elem(vfi_ctx* c, int kernel, const void* in0, const void* in1, const int32_t* f0, const int32_t* f1,
                           int n_frames, void* out, int C, int B, int H, int W, int h, int w, float slope, int which,
                           void* stream) {
  SepState* s = c ? ctx_sep(c) : nullptr;
  if (!s || !s->loaded) return sfail(VFI_E_STATE, "vfi_sepconv_load has not been called");
  if (kernel < 0 || kernel > 8) return sfail(VFI_E_INVALID, "sepconv: no such element-wise kernel");
  if (!in0 || !out || ((kernel == 1 || kernel == 8) && !in1)) return sfail(VFI_E_INVALID, "null argument");
  if (B < 1 || B > kMaxBatch) return sfail(VFI_E_INVALID, "sepconv: B must be in [1,16]");
  if (H < 1 || W < 1) return sfail(VFI_E_INVALID, "sepconv: empty launch");
  const bool frames = kernel == 0 || kernel == 1 || kernel == 7;
  SepPairIdx idx{};
  if (frames) {
    if (C < 3) return sfail(VFI_E_INVALID, "sepconv: frames need >= 3 channels");
    if (!f0 || !f1) return sfail(VFI_E_INVALID, "null argument");
    if (kernel == 7 && (which < 0 || which > 1)) return sfail(VFI_E_INVALID, "sepconv: pad_input pads frame 0 or 1");
    for (int i = 0; i < B; ++i) {
      if (f0[i] < 0 || f0[i] >= n_frames || f1[i] < 0 || f1[i] >= n_frames) return sfail(VFI_E_INVALID, "sepconv: frame index");
      idx.f0[i] = f0[i];
      idx.f1[i] = f1[i];
    }
  }
  if (kernel >= 2 && kernel <= 5 && (C < 8 || (C & 7))) return sfail(VFI_E_INVALID, "sepconv: C must be a multiple of 8");
  if ((kernel == 4 || kernel == 5) && (h < 1 || w < 1)) return sfail(VFI_E_INVALID, "sepconv: empty source");
  if (kernel == 4 && (H > 2 * h || W > 2 * w)) return sfail(VFI_E_INVALID, "sepconv: up-sampling target larger than 2h x 2w");
  if (kernel == 5 && (h < H || w < W)) return sfail(VFI_E_INVALID, "sepconv: crop source smaller than its target");
  const int op = s->op_type;
  const int He = H + (H & 1), We = W + (W & 1);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  SCK(cudaSetDevice(ctx_info(c).device));
  cudaError_t e = cudaSuccess;
  switch (kernel) {
    case 0:
      SCK(s->statp.ensure((size_t)B * sep_stats_blocks(He, We) * 2 * sizeof(double)));
      e = launch_sep_stats((const float*)in0, C, idx, B, H, W, He, We, (double*)out, (double*)s->statp.p, st);
      break;
    case 1:
      e = launch_sep_input_conv(op, (const float*)in0, C, idx, B, H, W, He, We, (const double*)in1, s->in_w, s->in_b,
                                s->enc_s0[1], out, st);
      break;
    case 2: e = launch_prelu_s2d16(op, in0, out, slope, C, B, H, W, st); break;
    case 3: e = launch_prelu16(op, in0, out, slope, (size_t)B * H * W * C, st); break;
    case 4: e = launch_prelu_up2_16(op, in0, out, slope, C, B, h, w, H, W, st); break;
    case 5: e = launch_add_crop16(op, in0, h, w, out, C, B, H, W, st); break;
    case 6: e = launch_sep_coeff_nchw(op, in0, 64, (float*)out, kK, B, H, W, st); break;
    case 7:
      e = launch_sep_pad_input((const float*)in0, C, idx, which, B, H, W, He + kK - 1, We + kK - 1, (float*)out, st);
      break;
    case 8: e = launch_sep_finish((const float*)in0, (const float*)in1, (float*)out, B, H, W, He, We, st); break;
  }
  ctx_add_launches(c, 1);
  if (e == cudaErrorInvalidValue) return sfail(VFI_E_INVALID, "sepconv: launch refused");
  if (e != cudaSuccess) return sfail(VFI_E_CUDA, std::string("sepconv: element-wise launch: ") + cudaGetErrorString(e));
  return VFI_OK;
}

/* Host-only: the packer of vfi_sepconv_load on caller data - a 3x3 conv [cout][cin][3][3] packed as a stride-1 layer
 * (stride2 = 0) or as the 2x2 conv over the space-to-depth input that runs its stride-2 form (stride2 = 1). */
int vfi_sepconv_debug_pack_host(int stride2, int cin, int cout, int n_total, int operand_type, const float* w, uint16_t* out,
                                int64_t out_cap, int* c0, int* n_cta, int* nsplit) {
  if (!w || !out) return sfail(VFI_E_INVALID, "null argument");
  StreamConvLayer L;
  L.ext = 1;
  L.n_total = n_total;
  L.ksize = stride2 ? 2 : 3;
  L.pad_before = stride2 ? 1 : -1;
  L.c0 = stride2 ? 4 * cin : cin;
  std::vector<uint16_t> pk;
  StreamConvParams p{};
  const bool ok = pack_streamconv(L, operand_type, [&](int n, int tap, int j) -> float {
    if (n >= cout) return 0.f;
    if (!stride2) return w[((size_t)n * cin + j) * 9 + tap];
    const int ab = j / cin, cc = j - ab * cin;
    const int ky = 2 * (tap >> 1) + (ab >> 1) - 1, kx = 2 * (tap & 1) + (ab & 1) - 1;
    if (ky < 0 || kx < 0) return 0.f;
    return w[((size_t)n * cin + cc) * 9 + ky * 3 + kx];
  }, &pk, &p);
  if (!ok) return sfail(VFI_E_INVALID, "sepconv: layer shape not supported by streamconv");
  if ((int64_t)pk.size() > out_cap) return sfail(VFI_E_INVALID, "output buffer too small");
  std::memcpy(out, pk.data(), pk.size() * 2);
  if (c0) *c0 = L.c0;
  if (n_cta) *n_cta = p.n_cta;
  if (nsplit) *nsplit = p.nsplit;
  return VFI_OK;
}

}  // extern "C"
