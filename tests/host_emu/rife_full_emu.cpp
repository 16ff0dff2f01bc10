// Whole-path host emulation of the RIFE path (TEST INFRASTRUCTURE): csrc/rife46.cu (context, weight repacking, the forward
// schedule, the host pipeline, the C ABI), csrc/elementwise.cu (prep / front / final / warp kernels) and csrc/tapconv.cu's
// plan + CUDA-core checker kernel, compiled for the host through cuda_shim_block.h.  The wgmma kernel is not emulated
// (launch_tapconv falls back to the checker with the same packed weights; wgmma vs checker is tests/test_gpu_layers.py).
#include "cuda_shim_block.h"

#include <string>

#include "../../comfyui-frame-interpolation_b200/csrc/vfi_internal.h"
namespace vfi {
// pieces of other translation units the C ABI in rife46.cu refers to but this emulation does not exercise
void film_destroy(FilmState*) {}
void sepconv_destroy(SepState*) {}
cudaError_t launch_softsplat_sum(const float*, const float*, float*, int, int, int, int, cudaStream_t) { return cudaErrorNotSupported; }
cudaError_t launch_softsplat_weighted(const float*, const float*, const float*, int, int, float*, float*, int, int, int, int, cudaStream_t) { return cudaErrorNotSupported; }
size_t ops_scratch_floats(int, int, int, int) { return 0; }
cudaError_t launch_softsplat_weighted_nhwc(const float*, const float*, const float*, int, int, float*, float*, float*, float*, int, int, int, int, cudaStream_t) { return cudaErrorNotSupported; }
cudaError_t launch_volume81_warp(bool, const float*, const float*, float*, float*, float*, int, int, int, int, cudaStream_t) { return cudaErrorNotSupported; }
cudaError_t launch_volume81(bool, const float*, const float*, float*, int, int, int, int, cudaStream_t) { return cudaErrorNotSupported; }
cudaError_t launch_sepconv(const float*, const float*, const float*, float*, int, int, int, int, int, int, cudaStream_t) { return cudaErrorNotSupported; }
cudaError_t launch_adacof(const float*, const float*, const float*, const float*, float*, int, int, int, int, int, int, int, int, cudaStream_t) { return cudaErrorNotSupported; }
cudaError_t launch_edt_pass(const float*, float*, int, int, int, float, cudaStream_t) { return cudaErrorNotSupported; }
}  // namespace vfi

#include "../../comfyui-frame-interpolation_b200/csrc/elementwise.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/tapconv.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/rife46.cu"
