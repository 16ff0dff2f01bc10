// Whole-path host emulation of the FILM path (TEST INFRASTRUCTURE): csrc/film.cu (weight loading / channel maps, the forward
// schedule of ~190 launches, buffer sizing, the C ABI), csrc/film_elem.cu and csrc/streamconv.cu's packer + CUDA-core
// checker kernel, compiled for the host through cuda_shim.h.  The wgmma kernel is not emulated (the checker stands in, as
// `vfi_film_debug_set_ref(ctx, 1)` selects on a GPU; wgmma vs checker is a GPU test).
#include "cuda_shim.h"

#include <string>

#include "../../comfyui-frame-interpolation_b200/csrc/vfi_internal.h"

struct vfi_ctx {
  vfi::FilmState* film = nullptr;
  int launches = 0;
};
namespace vfi {
static std::string g_err;
void set_error(const std::string& s) { g_err = s; }
CtxInfo ctx_info(::vfi_ctx*) { return CtxInfo{0, 132, nullptr, nullptr, nullptr}; }
FilmState*& ctx_film(::vfi_ctx* c) { return c->film; }
void ctx_add_launches(::vfi_ctx* c, int n) { c->launches += n; }
}  // namespace vfi
extern "C" const char* vfi_last_error(void) { return vfi::g_err.c_str(); }

#include "../../comfyui-frame-interpolation_b200/csrc/film_elem.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/streamconv.cu"
#include "../../comfyui-frame-interpolation_b200/csrc/film.cu"

extern "C" {
// a loaded context (operand_type: VFI_OPERAND_F16 / VFI_OPERAND_BF16) with every conv on the checker, for the C ABI's
// forward and test hooks (vfi_film_forward, vfi_film_debug_state, vfi_film_debug_elem); NULL on failure
vfi_ctx* emu_film_open(const float* const* tensors, const int64_t* numel, int n_tensors, int operand_type) {
  vfi_ctx* ctx = new vfi_ctx;
  if (vfi_film_load(ctx, tensors, numel, n_tensors, operand_type) || vfi_film_debug_set_ref(ctx, 1)) {
    vfi::film_destroy(ctx->film);
    delete ctx;
    return nullptr;
  }
  return ctx;
}
void emu_film_close(vfi_ctx* ctx) {
  vfi::film_destroy(ctx->film);
  delete ctx;
}

// flows (optional): the five finest levels of the forward, then of the backward flow pyramid, each [H_l, W_l, 2] fp32,
// concatenated (what debug_forward returns as forward_flow_pyramid / backward_flow_pyramid, film_arch.py:417-419, :450-455)
int emu_film(const float* const* tensors, const int64_t* numel, int n_tensors, const float* frames, int H, int W, int C,
             int clamp01, float* out, float* flows, int operand_type) {
  vfi_ctx ctx;
  int rc = vfi_film_load(&ctx, tensors, numel, n_tensors, operand_type);
  if (rc) return rc;
  rc = vfi_film_debug_set_ref(&ctx, 1);
  if (rc) return rc;
  const int32_t f0[1] = {0}, f1[1] = {1};
  rc = vfi_film_forward(&ctx, frames, 2, H, W, C, f0, f1, 1, clamp01, out, nullptr);
  if (!rc && flows) {
    float* dst = flows;
    for (int dir = 0; dir < 2; ++dir)
      for (int l = 0; l < 5; ++l) {
        const size_t n = (size_t)(H >> l) * (W >> l) * 2;
        std::memcpy(dst, ctx.film->v[dir][l].p, n * sizeof(float));
        dst += n;
      }
  }
  vfi::film_destroy(ctx.film);
  return rc ? rc : 1000 + ctx.launches;
}

// two pairs (frames 0-1 and 1-2) in ONE call: out [2, H, W, 3]
int emu_film_batch2(const float* const* tensors, const int64_t* numel, int n_tensors, const float* frames, int H, int W, int C,
                    float* out) {
  vfi_ctx ctx;
  int rc = vfi_film_load(&ctx, tensors, numel, n_tensors, VFI_OPERAND_F16);
  if (rc) return rc;
  rc = vfi_film_debug_set_ref(&ctx, 1);
  if (rc) return rc;
  const int32_t f0[2] = {0, 1}, f1[2] = {1, 2};
  rc = vfi_film_forward(&ctx, frames, 3, H, W, C, f0, f1, 2, 1, out, nullptr);
  vfi::film_destroy(ctx.film);
  return rc;
}
}
