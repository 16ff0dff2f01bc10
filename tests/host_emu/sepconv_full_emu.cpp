// Whole-path host emulation of the Sepconv trunk (TEST INFRASTRUCTURE): csrc/sepconv.cu (weight loading, the forward
// schedule, buffer sizing, the C ABI), csrc/sepconv_elem.cu and csrc/streamconv.cu's packer + CUDA-core checker kernel,
// and csrc/ops.cu's tiled separable-convolution kernel, compiled for the host through cuda_shim_block.h (blocks on host
// threads, threads as fibers).  What is NOT emulated: the wgmma kernel (the checker stands in, exactly as
// `vfi_sepconv_debug_set_ref(ctx, 1)` selects on a GPU).
#include "cuda_shim_block.h"

#include <string>

#include "../../comfyui-frame-interpolation_b200/csrc/vfi_internal.h"

struct vfi_ctx {
  vfi::SepState* sep = nullptr;
  int launches = 0;
};
namespace vfi {
static std::string g_err;
void set_error(const std::string& s) { g_err = s; }
CtxInfo ctx_info(::vfi_ctx*) { return CtxInfo{0, 132, nullptr, nullptr, nullptr}; }
SepState*& ctx_sep(::vfi_ctx* c) { return c->sep; }
void ctx_add_launches(::vfi_ctx* c, int n) { c->launches += n; }
}  // namespace vfi
extern "C" const char* vfi_last_error(void) { return vfi::g_err.c_str(); }

#include "../../comfyui-frame-interpolation_b200/csrc/ops.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/sepconv_elem.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/streamconv.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/sepconv.cu"

extern "C" {
// a loaded context (operand_type: VFI_OPERAND_F16 / VFI_OPERAND_BF16) with every conv on the checker, for the C ABI's
// forward and test hooks (vfi_sepconv_forward, vfi_sepconv_debug_state, vfi_sepconv_debug_elem); NULL on failure
vfi_ctx* emu_sepconv_open(const float* const* tensors, const int64_t* numel, int n_tensors, int operand_type) {
  vfi_ctx* ctx = new vfi_ctx;
  if (vfi_sepconv_load(ctx, tensors, numel, n_tensors, operand_type) || vfi_sepconv_debug_set_ref(ctx, 1)) {
    vfi::sepconv_destroy(ctx->sep);
    delete ctx;
    return nullptr;
  }
  return ctx;
}
void emu_sepconv_close(vfi_ctx* ctx) {
  vfi::sepconv_destroy(ctx->sep);
  delete ctx;
}
// the separable-convolution op (csrc/ops.cu, the launcher behind vfi_sepconv and the forward's two op launches)
int emu_sepconv_op(const float* in, const float* ver, const float* hor, float* out, int N, int C, int H, int W, int Kv, int Kh) {
  return (int)vfi::launch_sepconv(in, ver, hor, out, N, C, H, W, Kv, Kh, nullptr);
}

// weights in, one pair in, one frame out - everything through the product's own vfi_sepconv_load / vfi_sepconv_forward
// coef (optional): [4][51][He][We] fp32 = the coefficient planes of the heads Verone, Vertwo, Horone, Hortwo
int emu_sepconv(const float* const* tensors, const int64_t* numel, int n_tensors, const float* frames, int H, int W, int C,
                float* out, float* coef) {
  vfi_ctx ctx;
  int rc = vfi_sepconv_load(&ctx, tensors, numel, n_tensors, VFI_OPERAND_F16);
  if (rc) return rc;
  rc = vfi_sepconv_debug_set_ref(&ctx, 1);
  if (rc) return rc;
  const int32_t f0[1] = {0}, f1[1] = {1};
  rc = vfi_sepconv_forward(&ctx, frames, 2, H, W, C, f0, f1, 1, out, nullptr);
  if (!rc && coef) {
    const size_t n = (size_t)51 * (H + (H & 1)) * (W + (W & 1));
    for (int k = 0; k < 4; ++k) std::memcpy(coef + k * n, ctx.sep->coef[k].p, n * sizeof(float));
  }
  vfi::sepconv_destroy(ctx.sep);
  return rc ? rc : 1000 + ctx.launches;   // 1000 + number of launches on success
}

// several pairs of one clip in ONE call (the C ABI takes up to 16): frames [n_frames][H][W][C], pairs (f0[i], f1[i]),
// out [n_pairs][H][W][3]; 4-channel frames exercise the channel stride
int emu_sepconv_pairs(const float* const* tensors, const int64_t* numel, int n_tensors, const float* frames, int n_frames, int H,
                      int W, int C, const int32_t* f0, const int32_t* f1, int n_pairs, float* out) {
  vfi_ctx ctx;
  int rc = vfi_sepconv_load(&ctx, tensors, numel, n_tensors, VFI_OPERAND_F16);
  if (rc) return rc;
  rc = vfi_sepconv_debug_set_ref(&ctx, 1);
  if (rc) return rc;
  rc = vfi_sepconv_forward(&ctx, frames, n_frames, H, W, C, f0, f1, n_pairs, out, nullptr);
  vfi::sepconv_destroy(ctx.sep);
  return rc ? rc : 1000 + ctx.launches;
}
}
