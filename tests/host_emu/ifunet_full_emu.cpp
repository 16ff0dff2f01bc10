// Whole-path host emulation of the IFUnet path (TEST INFRASTRUCTURE): csrc/ifunet.cu (weight loading, BatchNorm
// folding and packing, the channel layout, the forward schedule, the workspace, the C ABI), csrc/ifunet_elem.cu,
// csrc/film_elem.cu's nearest x2 and csrc/streamconv.cu's packer + CUDA-core checker kernel, compiled for the host through
// cuda_shim.h.  The wgmma kernel is not emulated (the checker stands in, as `vfi_ifunet_debug_set_ref(ctx, 1)` selects
// on a GPU).
#include "cuda_shim.h"

#include <string>

#include "../../comfyui-frame-interpolation_b200/csrc/vfi_internal.h"

struct vfi_ctx {
  vfi::ModelState* ifunet = nullptr;
  int launches = 0;
};
namespace vfi {
static std::string g_err;
void set_error(const std::string& s) { g_err = s; }
CtxInfo ctx_info(::vfi_ctx*) { return CtxInfo{0, 132, nullptr, nullptr, nullptr}; }
ModelState*& ctx_ifunet(::vfi_ctx* c) { return c->ifunet; }
void ctx_add_launches(::vfi_ctx* c, int n) { c->launches += n; }
}  // namespace vfi
extern "C" const char* vfi_last_error(void) { return vfi::g_err.c_str(); }

#include "../../comfyui-frame-interpolation_b200/csrc/film_elem.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/ifunet_elem.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/streamconv.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/ifunet.cu"

extern "C" {
// one pair: img0, img1, out [3][H][W]; returns 1000 + launches, or the error code
int emu_ifunet(const float* const* tensors, const int64_t* numel, int n_tensors, const float* img0, const float* img1,
               int H, int W, double t, double scale, int ensemble, float* out) {
  vfi_ctx ctx;
  int rc = vfi_ifunet_load(&ctx, tensors, numel, n_tensors, VFI_OPERAND_F16);
  if (!rc) rc = vfi_ifunet_debug_set_ref(&ctx, 1);
  if (!rc) rc = vfi_ifunet_forward(&ctx, img0, img1, H, W, t, scale, ensemble, out, nullptr);
  delete ctx.ifunet;
  return rc ? rc : 1000 + ctx.launches;
}
}
