// Whole-path host emulation of the CAIN path (TEST INFRASTRUCTURE): csrc/cain.cu (weight loading and packing, the
// bordered layout, the forward schedule, buffer sizing, the C ABI), csrc/cain_elem.cu and csrc/streamconv.cu's packer +
// CUDA-core checker kernel, compiled for the host through cuda_shim.h.  The wgmma kernel is not emulated (the checker
// stands in, as `vfi_cain_debug_set_ref(ctx, 1)` selects on a GPU).
#include "cuda_shim.h"

#include <string>

#include "../../comfyui-frame-interpolation_b200/csrc/vfi_internal.h"

struct vfi_ctx {
  vfi::ModelState* cain = nullptr;
  int launches = 0;
};
namespace vfi {
static std::string g_err;
void set_error(const std::string& s) { g_err = s; }
CtxInfo ctx_info(::vfi_ctx*) { return CtxInfo{0, 132, nullptr, nullptr, nullptr}; }
ModelState*& ctx_cain(::vfi_ctx* c) { return c->cain; }
void ctx_add_launches(::vfi_ctx* c, int n) { c->launches += n; }
}  // namespace vfi
extern "C" const char* vfi_last_error(void) { return vfi::g_err.c_str(); }

#include "../../comfyui-frame-interpolation_b200/csrc/cain_elem.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/streamconv.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/cain.cu"

extern "C" {
// one pair: img0, img1, out [3][H][W]; returns 1000 + launches, or the error code
int emu_cain(const float* const* tensors, const int64_t* numel, int n_tensors, const float* img0, const float* img1,
             int H, int W, float* out) {
  vfi_ctx ctx;
  int rc = vfi_cain_load(&ctx, tensors, numel, n_tensors, VFI_OPERAND_F16);
  if (!rc) rc = vfi_cain_debug_set_ref(&ctx, 1);
  if (!rc) rc = vfi_cain_forward(&ctx, img0, img1, H, W, out, nullptr);
  delete ctx.cain;
  return rc ? rc : 1000 + ctx.launches;
}
}
