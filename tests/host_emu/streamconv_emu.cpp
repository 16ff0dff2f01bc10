// Host emulation of csrc/streamconv.cu alone (TEST INFRASTRUCTURE): the plan, the product packer, the launcher's argument
// checks and the CUDA-core checker kernel, reached through the C hooks vfi_streamconv_debug_conv (impl 1) and
// vfi_streamconv_plan, compiled for the host through cuda_shim.h.  The wgmma kernel is not emulated; device pointers are
// host pointers here.
#include "cuda_shim.h"

#include <string>

#include "../../comfyui-frame-interpolation_b200/csrc/vfi_internal.h"

namespace vfi {
static std::string g_err;
void set_error(const std::string& s) { g_err = s; }
}  // namespace vfi
extern "C" const char* vfi_last_error(void) { return vfi::g_err.c_str(); }

#include "../../comfyui-frame-interpolation_b200/csrc/streamconv.cu"
