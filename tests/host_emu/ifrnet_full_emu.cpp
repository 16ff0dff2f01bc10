// Whole-path host emulation of the IFRNet path (TEST INFRASTRUCTURE): csrc/ifrnet.cu (weight loading, the channel
// layout and the packing of the side-channel, space-to-depth and ConvT phase layers, the forward schedule, buffer sizing,
// the C ABI), csrc/ifrnet_elem.cu and csrc/streamconv.cu's packer + CUDA-core checker kernel, compiled for the host
// through cuda_shim.h.  The wgmma kernel is not emulated (the checker stands in, as `vfi_ifrnet_debug_set_ref(ctx, 1)`
// selects on a GPU).
#include "cuda_shim.h"

#include <string>

#include "../../comfyui-frame-interpolation_b200/csrc/vfi_internal.h"

struct vfi_ctx {
  vfi::ModelState* ifrnet = nullptr;
  int launches = 0;
};
namespace vfi {
static std::string g_err;
void set_error(const std::string& s) { g_err = s; }
CtxInfo ctx_info(::vfi_ctx*) { return CtxInfo{0, 132, nullptr, nullptr, nullptr}; }
ModelState*& ctx_ifrnet(::vfi_ctx* c) { return c->ifrnet; }
void ctx_add_launches(::vfi_ctx* c, int n) { c->launches += n; }
}  // namespace vfi
extern "C" const char* vfi_last_error(void) { return vfi::g_err.c_str(); }

#include "../../comfyui-frame-interpolation_b200/csrc/ifrnet_elem.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/streamconv.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/ifrnet.cu"

extern "C" {
// one pair: img0, img1, out [3][H][W]; returns 1000 + launches, or the error code; variant reports the loaded arch
int emu_ifrnet(const float* const* tensors, const int64_t* numel, int n_tensors, const float* img0, const float* img1,
               int H, int W, double t, double embt, float* out, int* variant) {
  vfi_ctx ctx;
  int rc = vfi_ifrnet_load(&ctx, tensors, numel, n_tensors, VFI_OPERAND_F16);
  if (!rc) rc = vfi_ifrnet_debug_set_ref(&ctx, 1);
  if (!rc) rc = vfi_ifrnet_info(&ctx, variant);
  if (!rc) rc = vfi_ifrnet_forward(&ctx, img0, img1, H, W, t, embt, out, nullptr);
  delete ctx.ifrnet;
  return rc ? rc : 1000 + ctx.launches;
}
}
