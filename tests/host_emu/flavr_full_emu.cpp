// Whole-path host emulation of the FLAVR path (TEST INFRASTRUCTURE): csrc/flavr.cu (weight loading and packing of the
// temporal, space-to-depth and transposed-phase layers, the forward schedule, buffer sizing, the C ABI), csrc/flavr_elem.cu
// and csrc/streamconv.cu's packer + CUDA-core checker kernel, compiled for the host through cuda_shim.h.  The wgmma kernel
// is not emulated (the checker stands in, as `vfi_flavr_debug_set_ref(ctx, 1)` selects on a GPU).
#include "cuda_shim.h"

#include <string>

#include "../../comfyui-frame-interpolation_b200/csrc/vfi_internal.h"

struct vfi_ctx {
  vfi::ModelState* flavr = nullptr;
  int launches = 0;
};
namespace vfi {
static std::string g_err;
void set_error(const std::string& s) { g_err = s; }
CtxInfo ctx_info(::vfi_ctx*) { return CtxInfo{0, 132, nullptr, nullptr, nullptr}; }
ModelState*& ctx_flavr(::vfi_ctx* c) { return c->flavr; }
void ctx_add_launches(::vfi_ctx* c, int n) { c->launches += n; }
}  // namespace vfi
extern "C" const char* vfi_last_error(void) { return vfi::g_err.c_str(); }

#include "../../comfyui-frame-interpolation_b200/csrc/flavr_elem.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/streamconv.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/flavr.cu"

extern "C" {
// n_windows windows, window k = frames first[k] .. first[k] + 3; out [n_windows, H, W, 3]; returns 1000 + launches,
// or the error code; n_outputs / enc_bias report what the loader detected
int emu_flavr(const float* const* tensors, const int64_t* numel, int n_tensors, const float* frames, int n_frames, int H,
              int W, int C, const int32_t* first, int n_windows, float* out, int* n_outputs, int* enc_bias) {
  vfi_ctx ctx;
  int rc = vfi_flavr_load(&ctx, tensors, numel, n_tensors, VFI_OPERAND_F16);
  if (!rc) rc = vfi_flavr_debug_set_ref(&ctx, 1);
  if (!rc) rc = vfi_flavr_info(&ctx, n_outputs, enc_bias);
  if (!rc) rc = vfi_flavr_forward(&ctx, frames, n_frames, H, W, C, first, n_windows, out, nullptr);
  delete ctx.flavr;
  return rc ? rc : 1000 + ctx.launches;
}
}
