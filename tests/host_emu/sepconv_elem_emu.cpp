// Host build of csrc/sepconv_elem.cu's kernels (see cuda_shim.h) with C entry points for ctypes.  16-bit tensors are fp16.
#include "cuda_shim.h"

#include "../../comfyui-frame-interpolation_b200/csrc/sepconv_elem.cu"

using namespace vfi;
static SepPairIdx pair01() {
  SepPairIdx i{};
  i.f0[0] = 0;
  i.f1[0] = 1;
  return i;
}

extern "C" {
void emu_stats(const float* frames, int cstride, int H, int W, int He, int We, double* stats) {
  double partial[2] = {0.0, 0.0};
  sep_stats_kernel(frames, cstride, pair01(), H, W, He, We, partial);
  sep_stats_sum_kernel(partial, 1, stats);
}
void emu_input_conv(const float* frames, int cstride, int H, int W, int He, int We, const double* stats, const float* w,
                    const float* bias, float slope, uint16_t* out) {
  sep_input_conv_kernel<__half>(frames, cstride, pair01(), H, W, He, We, stats, w, bias, slope, (__half*)out, 1);
}
void emu_prelu_s2d16(const uint16_t* in, uint16_t* out, float slope, int C, int B, int H, int W) {
  prelu_s2d16_kernel<__half>((const __half*)in, (__half*)out, slope, C / 8, B, H, W);
}
void emu_prelu16(const uint16_t* in, uint16_t* out, float slope, size_t n) {
  prelu16_kernel<__half>((const __half*)in, (__half*)out, slope, n / 8);
}
void emu_prelu_up2_16(const uint16_t* in, uint16_t* out, float slope, int C, int B, int h, int w, int Ht, int Wt) {
  prelu_up2_16_kernel<__half>((const __half*)in, (__half*)out, slope, C / 8, B, h, w, Ht, Wt);
}
void emu_add_crop16(const uint16_t* v, int Hv, int Wv, uint16_t* x, int C, int B, int H, int W) {
  add_crop16_kernel<__half>((const __half*)v, Hv, Wv, (__half*)x, C / 8, B, H, W);
}
void emu_coeff_nchw(const uint16_t* in, int pitch, float* out, int K, int B, int H, int W) {
  sep_coeff_nchw_kernel<__half>((const __half*)in, pitch, out, K, B, (size_t)H * W);
}
void emu_pad_input(const float* frames, int cstride, int which, int H, int W, int Hp, int Wp, float* out) {
  sep_pad_input_kernel(frames, cstride, pair01(), which, H, W, Hp, Wp, out, 1);
}
void emu_finish(const float* o1, const float* o2, float* out, int B, int H, int W, int He, int We) {
  sep_finish_kernel(o1, o2, out, B, H, W, He, We);
}
}
