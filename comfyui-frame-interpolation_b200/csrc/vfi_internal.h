// Internal declarations shared by the .cu files of libvfi_b200.so (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <functional>
#include <string>
#include <vector>

struct vfi_ctx;

// kernel launch; tests/host_emu/cuda_shim.h defines a host version (a plain call per grid row) before this header
#ifndef VFI_LAUNCH
#define VFI_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#endif
// a kernel's dynamic shared memory as an array of `type` (the host emulation points it at a per-block buffer)
#ifndef VFI_DYN_SMEM
#define VFI_DYN_SMEM(type, name) extern __shared__ type name[]
#endif

namespace vfi {

// ---------------------------------------------------------------------------------------------
// tap-list implicit GEMM ("tapconv"): every convolution of an IFBlock is expressed as
//   out[b, y, x, n] = epi( sum_e sum_{c < 16*nk16_e} in[b, y+dy_e, x+dx_e, 8*chunk0_e + c] * W_e[c, n] )
// on ONE spatial grid (input grid == output grid, zero outside).  Stride-2 convs read a
// space-to-depth input, the transposed conv writes a 4x4 sub-pixel patch per grid cell.
// ---------------------------------------------------------------------------------------------
enum EpiMode : int {
  EPI_BIAS_LRELU = 0,  // out = lrelu(acc + shift)                               (conv0.0, conv0.1)
  EPI_RESCONV = 1,     // out = lrelu(acc + shift + in[b,y,x,n])                 (ResConv; beta folded into W, shift=bias*beta)
  EPI_LASTCONV = 2,    // out5[b, 4y+py, 4x+px] = acc + shift, n = c5*16 + py*4+px (ConvT(4,2,1)+PixelShuffle(2))
  EPI_BIAS = 3,        // out = acc + shift, no activation                        (Head_417.cnn3)
};

struct TapEntry {
  int16_t dy, dx;   // spatial offset of this tap on the grid
  int16_t chunk0;   // first 8-channel chunk of the input it reads
  int16_t nk16;     // number of K=16 MMA steps (16 input channels each)
};

constexpr int kMaxTaps = 27;  // 9 taps, or 9 taps x 3 k-blocks in k-block-major order
constexpr int kTileH = 16, kTileW = 8;        // one CTA tile = 128 grid cells = two m64 wgmma row blocks
constexpr int kSmemLimit = 232448;            // 227 KB opt-in maximum per CTA on sm_90

constexpr int kMaxKBlocks = 6;
constexpr int kMaxK16 = 108;   // 9 taps x 192/16

struct alignas(64) TapConvParams {
  CUtensorMap tm64;      // input as a {C, W, H, B} tensor with a {64 ch, halo_w, halo_h, 1} box, SWIZZLE_128B
  CUtensorMap tm32;      // same with a {32 ch, ...} box, SWIZZLE_64B (only used when cin % 64 == 32)
  CUtensorMap tm_out;    // out_stage_bytes != 0: the output as {n_total, W, H, B}, box {store_box_c(n_cta), 8, 16, 1} (tapconv.cu)
  const void* in;        // [B, H, W, cin] 16-bit, NHWC
  void* out;             // [B, H, W, n_total] 16-bit NHWC; out_s2d = 1: its space-to-depth form; out_s2d = 2: the 4x4
                         // sub-pixel patch form [B, 4H, 4W, 8] with column n = (py*4 + px)*8 + ch (arch 4.26 lastconv features)
  float4* out_flow;      // EPI_LASTCONV: [B, 4H, 4W] float4 (4 flow components)
  float* out_mask;       // EPI_LASTCONV: [B, 4H, 4W]
  const void* w;         // packed weights: [nsplit][ceil(K16/4)][n_cta][128 B swizzled row] 16-bit
  const float* shift;    // [n_total]
  int B, H, W, cin;
  int n_total, n_cta, nsplit;
  int ntaps, ktotal16;
  int halo_y0, halo_x0, halo_h, halo_w;
  int stages;
  int epi_mode, out_s2d;
  int nruns, run_len;    // MMA issue: nruns runs of run_len consecutive K=16 steps (mma[r] = first step of run r)
  int cmajor;            // 1: channel-major MMAs, the 64 output channels on the wgmma M and the tile's 128 cells on N
  int wstream;           // 1: the weights stream through w_slots slots of four K=16 steps (see tapconv.cu)
  int w_slots, w_groups; //    slots in shared memory / slots per tile (ceil(K16 / 4))
  uint32_t w_slot_bytes; //    n_cta rows of 128 B
  int tiles_x, tiles_y, ntiles;
  int ctas_per_split;
  uint32_t b_hi;                  // high word of the weight (B) descriptors
  uint32_t w_bytes;               // packed weight bytes of one split
  uint32_t off_w, off_a, stage_bytes, smem_bytes;
  uint32_t off_out, out_stage_bytes;  // per-warpgroup staging tiles of the TMA output stores (0: direct stores)
  int nkb;                        // k-blocks of the staged window: 64 channels each, 32-channel tail if cin%64==32
  uint32_t kb_off[kMaxKBlocks];   // byte offset of each k-block inside a stage (1024-aligned)
  uint32_t tx_bytes;              // bytes one stage fill delivers (mbarrier transaction count)
  TapEntry taps[kMaxTaps];
  // per run: {A start offset inside a stage, A descriptor high word, B start offset inside the weights, 0},
  // offsets in 16-byte units.  Lives in the kernel parameters (constant bank): uniform loads for the MMA warpgroups.
  uint4 mma[kMaxK16];
};

// A convolution layer bound to its packed weights.
struct TapConvLayer {
  int cin = 0, n_total = 0, n_cta = 0, nsplit = 1;
  int ntaps = 0, ktotal16 = 0;
  int halo_y0 = 0, halo_x0 = 0, halo_h = 0, halo_w = 0;
  int epi_mode = 0, out_s2d = 0;
  int wstream = 0;        // streamed weights, whole window per tile (the ResConvs of blocks 0-2, block 1's lastconv
                          // and the 4.26 feature conv of blocks 0 and 1; see tapconv.cu)
  TapEntry taps[kMaxTaps];
  void* w = nullptr;      // device
  float* shift = nullptr; // device
};

struct BatchTasks {       // passed by value to the full-resolution kernels
  int n;
  int f0[16];
  int f1[16];
  float t[16];
};
constexpr int kMaxBatch = 16;

// operand element type of the tensor-core path
enum OperandType : int { OP_F16 = 0, OP_BF16 = 1 };

// ---- launchers (defined in tapconv.cu / elementwise.cu) -------------------------------------
// Returns cudaSuccess or the launch error.  impl: 0 the tensor-core kernel as planned, 1 the CUDA-core checker, 2 the
// tensor-core kernel with cells on the wgmma M even where the plan chose the channel-major MMAs (A/B comparisons).
enum TapConvImpl : int { TAPCONV_PLANNED = 0, TAPCONV_CHECKER = 1, TAPCONV_CELL_MAJOR = 2 };
cudaError_t launch_tapconv(const TapConvLayer& L, int op_type, const void* in, void* out, float4* out_flow,
                           float* out_mask, int B, int H, int W, int num_sms, int impl, cudaStream_t st);
// smem/stage plan for a layer (for DESIGN.md tables and tests); returns 0 stages when it cannot fit
int tapconv_plan(const TapConvLayer& L, TapConvParams* p_out);
// conv0.0 (L0) and conv0.1 (L1) of a 64-channel arch-4.6 IFBlock as one launch (tapconv.cu): x [B, H, W, 64] -> out
// [B, H/2, W/2, 64], conv0.0's output kept in shared memory.  The host emulation runs the two checker launches through
// c00 instead.  conv0_fused_plan returns its x window stages (0: the pair is not of that shape) and its shared-memory
// bytes, registers per thread and local (spill) bytes per thread.
int conv0_fused_plan(const TapConvLayer& L0, const TapConvLayer& L1, int op_type, int* smem_bytes, int* regs,
                     int* local_bytes);
cudaError_t launch_conv0_fused(const TapConvLayer& L0, const TapConvLayer& L1, int op_type, const void* x, void* c00,
                               void* out, int B, int H, int W, int num_sms, cudaStream_t st);

// imgs: fp32 float4 planes (final blend); imgs_h: the same pixels as half4 (8 bytes) for the block-input warps, whose
// results are rounded to 16 bits anyway - half the gather bytes through L1
cudaError_t launch_prep_frames(const float* frames, int n, int H, int W, int cstride, float4* imgs, uint2* imgs_h,
                               int Hp, int Wp, cudaStream_t st);
// low-resolution outputs of the blocks executed so far (the accumulated full-resolution flow is implicit)
constexpr int kMaxBlocks = 5;  // arch 4.26 has five IFBlocks, the others four
struct FlowState {
  float4* f[kMaxBlocks];
  float* m[kMaxBlocks];
  int s[kMaxBlocks];
  int n;             // number of blocks
  int mask_replace;  // arch 4.7+: mask = newest level only
};
cudaError_t launch_encode(const float4* imgs, const float* w0, const float* b0, const float* w1, const float* b1,
                          float* e16, uint2* feats, int n, int Hp, int Wp, cudaStream_t st);
cudaError_t launch_head0(int op_type, const float4* imgs, const float* w, const float* bias, void* out, int n, int Hp,
                         int Wp, cudaStream_t st);
// arch 46, 47, 417 or 426.  feats: arch 4.7 half4 planes, arch 4.17 / 4.26 16-bit space-to-depth planes of 8 / 4
// channels, or nullptr (4.6).  prev_feat: arch 4.26, blocks > 0: the previous block's 8 lastconv feature channels
// [B, Hp/prev_s, Wp/prev_s, 8] 16-bit.
cudaError_t launch_front(int op_type, int arch, const float4* imgs, const uint2* imgs_h, const void* feats,
                         const void* prev_feat, int prev_s, const FlowState& fs, int blk, int lo,
                         const float4* base_f, const float* base_m, float4* out_f, float* out_m, BatchTasks tasks,
                         int Hp, int Wp, int s, void* x_s2d, cudaStream_t st);
// (launch_materialize / launch_final add levels [lo, fs.n) to the base)
cudaError_t launch_materialize(const FlowState& fs, int lo, const float4* base_f, const float* base_m, float4* flow,
                               float* mask, int B, int Hp, int Wp, cudaStream_t st);
cudaError_t launch_final(const float4* imgs, const FlowState& fs, int lo, const float4* base_f, const float* base_m,
                         BatchTasks tasks, int Hp, int Wp, int H, int W, float* out, cudaStream_t st);
// up-scaled blocks (scale_factor 2 / 4): block input k times finer than full resolution from the dense planes,
// and the block's output folded back onto them
cudaError_t launch_front_up(int op_type, int arch, const uint2* imgs_h, const void* feats, const void* prev_feat, int prev_s,
                            int prev_k, const float4* F, const float* M, BatchTasks tasks, int Hp, int Wp, int k, void* x_s2d,
                            cudaStream_t st);
cudaError_t launch_fold_down(const float4* tf, const float* tm, int k, float4* F, float* M, int B, int Hp, int Wp,
                             int mask_replace, cudaStream_t st);
cudaError_t launch_warp(const float* img, const float* flow, float* out, int B, int H, int W, int C, cudaStream_t st);

cudaError_t launch_softsplat_sum(const float* in, const float* flow, float* out, int N, int C, int H, int W,
                                 cudaStream_t st);
cudaError_t launch_softsplat_weighted(const float* in, const float* flow, const float* metric, int mode, int eps, float* out,
                                      float* norm, int N, int C, int H, int W, cudaStream_t st);
// channel-last forms (ops.cu): NCHW in / out like the forms above, `sa` / `sb` = scratch of ops_scratch_floats() floats each
size_t ops_scratch_floats(int N, int C, int H, int W);
cudaError_t launch_softsplat_weighted_nhwc(const float* in, const float* flow, const float* metric, int mode, int eps, float* out,
                                           float* norm, float* sa, float* sb, int N, int C, int H, int W, cudaStream_t st);
cudaError_t launch_volume81_warp(bool dot, const float* one, const float* two, float* out, float* sa, float* sb, int N, int C, int H,
                                 int W, cudaStream_t st);
cudaError_t launch_volume81(bool dot, const float* one, const float* two, float* out, int N, int C, int H, int W,
                            cudaStream_t st);
cudaError_t launch_sepconv(const float* in, const float* ver, const float* hor, float* out, int N, int C, int H, int W,
                           int Kv, int Kh, cudaStream_t st);


// ---------------------------------------------------------------------------------------------
// streamconv (streamconv.cu): k x k 'same' convolution with streamed weights - the FILM conv kernel.
//   out[b, y, x, n] = act( bias[n] + sum_{tap, c} in[b, y+dy, x+dx, c] * W[tap, c, n] ),  in = cat(src0[:c0], src1[:c1])
// With kt > 1 it is a kt x k x k 3-D convolution over [sample][plane][H][W][C] tensors (FLAVR, flavr.cu): output plane t
// sums temporal taps dt = 0 .. kt-1 of input plane t + dt - pad_t (zero outside [0, T_in)).
// ---------------------------------------------------------------------------------------------
struct StreamConvLayer {
  int ksize = 3;          // 1, 2 or 3; padding='same' (film_arch.py:784-790)
  int c0 = 0, c1 = 0;     // input channels taken from source 0 / source 1 (multiples of 64; c1 may be 0)
  int n_total = 0;        // output channels (multiple of 16; padded with zero weights where the layer has fewer)
  int act = 1;            // 1: LeakyReLU(0.2), 0: none
  int ext = 0;            // 1: Sepconv epilogue instead: PReLU with one learned `slope` (1.0 = none), then + residual
                          // 2: IFRNet epilogue: + residual, then PReLU with per-channel `slopes`; columns < n_f32 fp32
  float slope = 1.f;
  const float* slopes = nullptr;  // ext 2: device, [n_total] PReLU slopes (1.0 = identity)
  int n_f32 = 0;                  // ext 2: output columns [0, n_f32) go to the fp32 tensor of the launch
  int pad_before = -1;    // rows / columns of zero padding before the window; -1: (ksize - 1) / 2 ('same')
  int pad_before_x = -1;  // columns of zero padding before the window when >= 0 (rows keep pad_before)
  int kt = 1, pad_t = 0;  // temporal taps and zero planes before plane 0
  int T_in = 1, T_out = 1;  // planes per sample of the input / output (the launch's B counts samples)
  void* w = nullptr;      // device, packed [split][dt][k-block][tap][n_cta][64 ch, 16-byte chunks XOR (n & 7)] 16-bit
  float* shift = nullptr; // device, [n_total] bias
};

struct alignas(64) StreamConvParams {
  CUtensorMap tm[2];      // sources as {C, W, H, B} tensors, box {64, halo_w, halo_h, 1}, SWIZZLE_128B
  const void* src[2];     // (checker kernel) source pointers and pixel pitches in elements
  int src_pitch[2];
  void* out;              // 16-bit NHWC, channel 0 of this layer's slice
  int out_pitch;          // elements per pixel of the output tensor
  const void* res;        // ext: residual added after (ext 2: before) the activation (layout of `out`), or nullptr
  float slope;            // ext 1: PReLU slope
  int ext;
  const float* slopes;    // ext 2: per-channel PReLU slopes [n_total]
  float* out_f32;         // ext 2: fp32 NHWC tensor of the columns [0, n_f32), pixel pitch f32_pitch
  int f32_pitch, n_f32;
  const void* w;
  const float* shift;
  size_t w_split_bytes;   // packed weight bytes of one output-channel split
  int B, H, W;            // B: output images (samples x T_out)
  int B_in;               // input images (samples x T_in)
  int kt, pad_t, T_in, T_out;
  int ksize, ntaps, nkb0, nkb;
  int n_total, n_cta, nsplit, act;
  int halo_y0, halo_x0, halo_h, halo_w;
  int mt;                 // tiles per CTA pass (one per MMA warpgroup, sharing every weight slot)
  int a_slots, b_slots;
  int tiles_x, tiles_y, ntiles, npasses, ctas_per_split;
  uint32_t a_tx_bytes, a_win_bytes, a_slot_bytes, b_slot_bytes;
  uint32_t off_b, off_a, smem_bytes;
  uint32_t a_hi;          // high word of the A descriptors
  uint32_t tap_off[9];    // start-address offset of each tap inside a window, 16-byte units
};

bool streamconv_plan(const StreamConvLayer& L, StreamConvParams* p_out);
cudaError_t launch_streamconv(const StreamConvLayer& L, int op_type, const void* src0, int pitch0, const void* src1,
                              int pitch1, void* out, int out_pitch, int B, int H, int W, int num_sms, bool use_ref,
                              cudaStream_t st, const void* res = nullptr, float* out_f32 = nullptr, int f32_pitch = 0);

// host-only operand packer (film.cu): wfun(output column n, tap = ky * k + kx, padded input channel) -> weight
bool pack_streamconv(const StreamConvLayer& L, int op_type, const std::function<float(int, int, int)>& wfun,
                     std::vector<uint16_t>* out, StreamConvParams* plan);
// the same with temporal taps (flavr.cu): wfun(output column n, temporal tap dt, tap, padded input channel) -> weight
bool pack_streamconv3d(const StreamConvLayer& L, int op_type, const std::function<float(int, int, int, int)>& wfun,
                       std::vector<uint16_t>* out, StreamConvParams* plan);

// ---- Sepconv element-wise kernels (sepconv_elem.cu) ----
struct SepPairIdx {  // source frames of every pair of a pass
  int f0[16];
  int f1[16];
};
struct SepState;
void sepconv_destroy(SepState* s);  // sepconv.cu
// stats [B, 2]; partial: scratch of B * sep_stats_blocks(He, We) * 2 doubles
int sep_stats_blocks(int He, int We);
cudaError_t launch_sep_stats(const float* frames, int cstride, const SepPairIdx& idx, int B, int H, int W, int He, int We,
                             double* stats, double* partial, cudaStream_t st);
cudaError_t launch_sep_input_conv(int op, const float* frames, int cstride, const SepPairIdx& idx, int B, int H, int W, int He,
                                  int We, const double* stats, const float* w, const float* bias, float slope, void* out,
                                  cudaStream_t st);
cudaError_t launch_prelu_s2d16(int op, const void* in, void* out, float slope, int C, int B, int H, int W, cudaStream_t st);
cudaError_t launch_prelu16(int op, const void* in, void* out, float slope, size_t n, cudaStream_t st);
cudaError_t launch_prelu_up2_16(int op, const void* in, void* out, float slope, int C, int B, int h, int w, int Ht, int Wt,
                                cudaStream_t st);
cudaError_t launch_add_crop16(int op, const void* v, int Hv, int Wv, void* x, int C, int B, int H, int W, cudaStream_t st);
cudaError_t launch_sep_coeff_nchw(int op, const void* in, int pitch, float* out, int K, int B, int H, int W, cudaStream_t st);
cudaError_t launch_sep_pad_input(const float* frames, int cstride, const SepPairIdx& idx, int which, int B, int H, int W,
                                 int Hp, int Wp, float* out, cudaStream_t st);
cudaError_t launch_sep_finish(const float* o1, const float* o2, float* out, int B, int H, int W, int He, int We,
                              cudaStream_t st);

// ---- FILM element-wise kernels (film_elem.cu); 16-bit tensors are NHWC slices {pointer, pixel pitch in elements} ----
struct FilmFrameIdx {  // source frame of every image of a pass (first frames of all pairs, then second frames)
  int i[2 * 16];
};
cudaError_t launch_film_gather_rgb(const float* frames, int cstride, const FilmFrameIdx& idx, int n, int H, int W,
                                   float* out, cudaStream_t st);
cudaError_t launch_film_pool_rgb(const float* in, float* out, int n, int H, int W, cudaStream_t st);
cudaError_t launch_film_conv_rgb(int op_type, const float* img, const float* w, const float* bias, void* out,
                                 int out_pitch, int n, int H, int W, cudaStream_t st);
cudaError_t launch_film_pool16(int op_type, const void* in, int in_pitch, void* out, int out_pitch, int C, int n, int H,
                               int W, cudaStream_t st);
cudaError_t launch_film_flow_up(const float* v, int h, int w, float* out, int B, int H, int W, cudaStream_t st);
cudaError_t launch_film_warp16(int op_type, const void* src, int src_pitch, int C, const float* flow, float fscale,
                               void* dst, int dst_pitch, int B, int H, int W, cudaStream_t st);
cudaError_t launch_film_misc64(int op_type, const float* img0, const float* img1, const float* bflow,
                               const float* fflow, void* dst, int dst_pitch, int B, int H, int W, cudaStream_t st);
cudaError_t launch_film_nearest16(const void* in, int h, int w, void* out, int C, int B, int H, int W, cudaStream_t st);
cudaError_t launch_film_flow_head(int op_type, const void* x, int pitch, int C, const float* w, const float* bias,
                                  const float* v_up, float* v_out, int B, int H, int W, cudaStream_t st);
cudaError_t launch_film_out_rgb(int op_type, const void* x, int pitch, const float* w, const float* bias, int clamp01,
                                float* out, int B, int H, int W, cudaStream_t st);

// ---- FLAVR kernels around the convolutions (flavr_elem.cu); images = windows x 4 planes ----
constexpr int kFlavrMaxWindows = 8;
struct FlavrFrameIdx {  // source frame of every image of a pass (window k, plane t at k * 4 + t)
  int i[4 * kFlavrMaxWindows];
};
cudaError_t launch_flavr_frame_sums(const float* frames, int cstride, const FlavrFrameIdx& idx, int n_img, int H, int W,
                                    int Hp, int Wp, int pt, int pl, float* sums, cudaStream_t st);
cudaError_t launch_flavr_prep(const float* frames, int cstride, const FlavrFrameIdx& idx, int n_img, int T, int H, int W,
                              int Hp, int Wp, int pt, int pl, const float* sums, float4* out, cudaStream_t st);
cudaError_t launch_flavr_stem(int op_type, const float4* xin, int n_img, int T, int Hp, int Wp, const float* w,
                              const float* bias, void* out, cudaStream_t st);
int flavr_sum_chunks(size_t npx);  // partial sums per sample of chan_sums (a function of the geometry only)
cudaError_t launch_flavr_chan_sums(int op_type, const void* x, int C, size_t npx, int S, float* partial, cudaStream_t st);
cudaError_t launch_flavr_gate(const float* partial, size_t npx, int groups, int C, size_t count, const float* w,
                              const float* b, int S, float* g, cudaStream_t st);
cudaError_t launch_flavr_apply(int op_type, const void* x, int phases, const float* g, const void* res, int act, void* out,
                               void* s2d, int C, int n_img, int T, int H, int W, cudaStream_t st);
cudaError_t launch_flavr_outconv(int op_type, const void* x, int S, int Hp, int Wp, int H, int W, int pt, int pl,
                                 const float* w, const float* bias, const float* sums, int T, float* out, cudaStream_t st);

// ---- IFRNet kernels around the convolutions (ifrnet_elem.cu); frames and output are fp32 [3][H][W] planes ----
int ifrnet_sum_blocks();  // partial sums of launch_ifrnet_mean (doubles)
cudaError_t launch_ifrnet_mean(const float* f0, const float* f1, int H, int W, int Hp, int Wp, double* partial, float* mean,
                               cudaStream_t st);
cudaError_t launch_ifrnet_prep(const float* f0, const float* f1, int H, int W, int Hp, int Wp, int h0, int w0, float scale,
                               const float* mean, float4* out, cudaStream_t st);
cudaError_t launch_ifrnet_first_conv(int op, const float4* xin, int h0, int w0, int h1, int w1, int k, const float* w,
                                     const float* bias, const float* slopes, int C, int pitch, void* out, cudaStream_t st);
cudaError_t launch_ifrnet_s2d(int op, const void* in, int pitch, int cq, int B, int h, int w, void* out, int opitch,
                              cudaStream_t st);
cudaError_t launch_ifrnet_dec4_in(int op, const void* f, int fpitch, int g1, int h, int w, float embt, void* out,
                                  cudaStream_t st);
cudaError_t launch_ifrnet_dec_flow(const float* ph, int nf, const float* prev, int h, int w, float* acc, cudaStream_t st);
cudaError_t launch_ifrnet_dec_in(int op, const void* ph16, int pp, const void* f, int fpitch, int fh, int fw,
                                 const float* acc, int gh, int gw, int g1, int g2, int g3, void* out, cudaStream_t st);
cudaError_t launch_ifrnet_final(const float* f0, const float* f1, int H, int W, int Hp, int Wp, const float* acc, int hq,
                                int wq, int hF, int wF, float scale, float fmul, const float* mean, float* out,
                                cudaStream_t st);

// ---- CAIN kernels around the convolutions (cain_elem.cu); 16-bit tensors on the bordered (h + 2) x (w + 2) grid,
// 192 channels per cell (the prep output 384); frames and output are fp32 [3][H][W] planes ----
constexpr int kCainChannels = 192;   // trunk channels (3 x 4^3)
constexpr int kCainMeanChunks = 64;  // partial sums per frame plane (doubles: 6 x kCainMeanChunks)
constexpr int kCainHidden = 12;      // CALayer's 192 / 16
cudaError_t launch_cain_frame_sums(const float* f0, const float* f1, int H, int W, double* partial, cudaStream_t st);
cudaError_t launch_cain_prep(int op, const float* f0, const float* f1, int H, int W, int top, int left, int h, int w,
                             const double* partial, void* out, cudaStream_t st);
// reflect: border = ReflectionPad2d(1) of the interior (add must be null); else border = 0 and interior += add (if any)
cudaError_t launch_cain_border(int op, void* x, const void* add, int h, int w, bool reflect, cudaStream_t st);
cudaError_t launch_cain_chan_sums(int op, const void* x, int h, int w, float* partial, cudaStream_t st);  // [h][192]
cudaError_t launch_cain_gate(const float* partial, int h, int w, const float* ca, float* g, cudaStream_t st);
cudaError_t launch_cain_apply(int op, const void* x, const float* g, const void* res, void* out, int h, int w,
                              cudaStream_t st);
cudaError_t launch_cain_final(int op, const void* feat, int H, int W, int top, int left, int w, const double* partial,
                              float* out, cudaStream_t st);

// ---- IFUnet kernels around the convolutions (ifunet_elem.cu); frames and output are fp32 [3][H][W] planes, padded
// frames (Hp x Wp) read zeros beyond H x W; 16-bit tensors NHWC; flows fp32 ----
constexpr int kIfuPoolChunks = 32;  // CBAM pool partials per image (a function of nothing but this constant)
struct IfuFlowIn {                  // one IFUNet level input (launch_ifunet_flow_in)
  const float* f0;
  const float* f1;
  int H, W, Hp, Wp;
  const float* warped;  // [2][3][Hp][Wp] fp32, or null at level 0
  const float* flow;    // [Hp][Wp][4] fp32, or null at level 0
  int swap0;            // batch image 0 reads (img1, img0, 1 - t); image 1 always the opposite of image 0
  float t;
  int resize;           // scale != 1
  float cscale, fscale; // coordinate scale (float)(1 / scale) and flow multiplier (float) scale
  int h0, w0;           // the resized input's size
  const float* c0w;     // level 0: conv0 weights [17][7], bias, PReLU slopes
  const float* c0b;
  const float* c0s;
};
cudaError_t launch_ifunet_flow_in(int op, const IfuFlowIn& a, int B, void* out, cudaStream_t st);
cudaError_t launch_ifunet_s2d(int op, const void* in, int pitch, int cq, int B, int h, int w, void* out, int opitch,
                              cudaStream_t st);
cudaError_t launch_ifunet_d2s(const void* ph, int C, int B, int h, int w, void* out, cudaStream_t st);
// CBAM in place on x [B][h][w][pitch] (C channels): mlp = {W1 [C/16][C], b1, W2 [C][C/16], b2}, sw = {7x7 weights
// [2][49], bias} with BatchNorm folded; scratch psum / pmax [B][kIfuPoolChunks][C], gate [B][C], cmp [B][h][w][2]
cudaError_t launch_ifunet_cbam(int op, void* x, int pitch, int C, int B, int h, int w, const float* mlp, const float* sw,
                               float* psum, float* pmax, float* gate, float* cmp, cudaStream_t st);
cudaError_t launch_ifunet_add16(int op, void* x, const void* y, size_t n, cudaStream_t st);
cudaError_t launch_ifunet_convex(int op, const float* flow, const void* mask, int L, int B, int h, int w, float* up,
                                 cudaStream_t st);
cudaError_t launch_ifunet_flow_update(const float* up, int uh, int uw, int resize, float cscale, float fmul, int mode,
                                      int Hp, int Wp, float* flow, cudaStream_t st);
cudaError_t launch_ifunet_warp_frames(const float* f0, const float* f1, int H, int W, int Hp, int Wp, const float* flow,
                                      float* warped, cudaStream_t st);
cudaError_t launch_ifunet_fusion_in(int op, const float* f0, const float* f1, int H, int W, int Hp, int Wp,
                                    const float* warped, const float* flow, void* out, cudaStream_t st);
cudaError_t launch_ifunet_rrdb_res(int op, void* y, const void* x, size_t n, cudaStream_t st);
cudaError_t launch_ifunet_merge(const float* warped, const float* last, int Hp, int Wp, float* deg, cudaStream_t st);
cudaError_t launch_ifunet_fb_in(const float* f0, const float* f1, int H, int W, int Hp, int Wp, const float* deg,
                                const float* rwarp, const float* rmask, const float* rflow, int cin, int s, float* out,
                                cudaStream_t st);
cudaError_t launch_ifunet_stem(int op, const float* src0, const float* src1, int cin, int sh, int sw, int vh, int vw,
                               const float* w, const float* bias, const float* slopes, int cout, int B, int pitch, void* out,
                               cudaStream_t st);
cudaError_t launch_ifunet_fb_out(const float* ph, int h, int w, int s, int first, const float* f0, const float* f1, int H,
                                 int W, int Hp, int Wp, float* rflow, float* rmask, float* rwarp, cudaStream_t st);
cudaError_t launch_ifunet_ctx_warp(int op, const void* feat, int fpitch, const float* rflow, int Hp, int Wp, void* out,
                                   cudaStream_t st);
cudaError_t launch_ifunet_final(const float* ph, const float* rwarp, const float* rmask, const float* deg, int H, int W,
                                int Hp, int Wp, float* out, cudaStream_t st);

cudaError_t launch_adacof(const float* in, const float* weight, const float* off_i, const float* off_j, float* out, int N,
                          int C, int Hin, int Win, int F, int dil, int Ho, int Wo, cudaStream_t st);
cudaError_t launch_edt_pass(const float* data, float* out, int bs, int h, int w, float diam2, cudaStream_t st);

void set_error(const std::string& s);

// ---- context access for film.cu (vfi_ctx is defined in rife46.cu) ----
struct FilmState;
// state that a model's .cu file keeps in a context; vfi_destroy deletes it through this base
struct ModelState {
  virtual ~ModelState() = default;
};
struct CtxInfo {
  int device, num_sms;
  cudaStream_t s_h2d, s_comp, s_d2h;
};
void film_destroy(FilmState* f);  // film.cu


CtxInfo ctx_info(::vfi_ctx* c);
FilmState*& ctx_film(::vfi_ctx* c);
ModelState*& ctx_flavr(::vfi_ctx* c);  // a FlavrState (flavr.cu)
ModelState*& ctx_ifrnet(::vfi_ctx* c);  // an IfrnetState (ifrnet.cu)
ModelState*& ctx_cain(::vfi_ctx* c);    // a CainState (cain.cu)
ModelState*& ctx_ifunet(::vfi_ctx* c);  // an IfunetState (ifunet.cu)
SepState*& ctx_sep(::vfi_ctx* c);
void ctx_add_launches(::vfi_ctx* c, int n);

}  // namespace vfi
