/* libvfi_b200.so - C ABI of the H100-native frame-interpolation hot path (RIFE 4.6 first).
 *
 * The reference (Fannovel16/ComfyUI-Frame-Interpolation @ 26545cc) has no native library: its "FFI" is
 * (a) PyTorch ATen calls from vfi_models/rife/rife_arch.py and (b) cupy RawModule launches that pass
 * `(int32 n, raw device pointers...)` on torch's current stream (vfi_models/ops/cupy_ops/softsplat.py:206-224).
 * This header is what a maintainer binds instead (ctypes stub in INTEGRATION.md).  Conventions:
 *   - plain pointers and sizes only, no torch types; device pointers are owned by the caller (PyTorch);
 *   - every function returns 0 on success or a negative VFI_E_* code; vfi_last_error() gives the text
 *     (thread-local);  the Python host raises RuntimeError, mirroring the reference's exception behaviour;
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream); no hidden synchronisation
 *     unless the function name says *_host or *_sync;
 *   - images are float32 NHWC in [0,1] exactly as ComfyUI's IMAGE type (rife/__init__.py:146,239).
 */
#ifndef VFI_B200_H
#define VFI_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VFI_OK 0
#define VFI_E_INVALID (-1)   /* bad argument / unsupported configuration */
#define VFI_E_CUDA (-2)      /* CUDA runtime or kernel error */
#define VFI_E_STATE (-3)     /* e.g. forward before weights were loaded */
#define VFI_E_NOTIMPL (-4)

#define VFI_OPERAND_F16 0    /* conv operands fp16, fp32 accumulate (node dtype float32 / float16) */
#define VFI_OPERAND_BF16 1   /* conv operands bf16, fp32 accumulate (node dtype bfloat16) */

#define VFI_RIFE46_NUM_TENSORS 120   /* IFNet("4.6").state_dict() - rife_arch.py:404-408 */
#define VFI_RIFE47_NUM_TENSORS 124   /* IFNet("4.7"): + encode.{0,1}.{weight,bias} - rife_arch.py:409-417 */
#define VFI_RIFE417_NUM_TENSORS 128  /* + encode.cnn0..cnn3 weight, bias (Head_417, rife_arch.py:356-363) */
#define VFI_RIFE426_NUM_TENSORS 158  /* IFNet("4.26"): 5 blocks x 30 + Head cnn0..cnn3 weight, bias (rife_arch.py:453-459) */
#define VFI_MAX_BATCH 16

typedef struct vfi_ctx vfi_ctx;

/* library / context ------------------------------------------------------------------------------------ */
const char* vfi_last_error(void);
const char* vfi_version(void);
/* Creates a context bound to CUDA device `device` (its own compute/copy streams, workspace, weights). */
int vfi_create(int device, vfi_ctx** out);
int vfi_destroy(vfi_ctx* ctx);
/* Number of kernels this library has launched through `ctx` since creation (bench.py "gpu_launches"). */
int64_t vfi_launch_count(const vfi_ctx* ctx);
/* Pairs interpolated per internal pass (1..VFI_MAX_BATCH, default 8); replaces the node's batch_size knob
 * (rife/__init__.py:64-69) - it changes scheduling only, never results. */
int vfi_set_batch(vfi_ctx* ctx, int batch);

/* Replaces: IFNet(arch_ver="4.6").load_state_dict(torch.load(path)) - rife/__init__.py:129-133.
 * `tensors[i]` are HOST float32 arrays in state_dict order (block{b}.conv0.0.0.weight, .bias, conv0.1.0.weight,
 * .bias, 8 x convblock.{j}.{beta, conv.weight, conv.bias}, lastconv.0.weight, .bias; b = 0..3); `numel[i]` is
 * checked against the architecture.  Weights are repacked to the tensor-core operand layout on the device. */
int vfi_rife46_load(vfi_ctx* ctx, const float* const* tensors, const int64_t* numel, int n_tensors, int operand_type);
/* Same for any built arch: 46 (rife46.pth), 47 (rife47.pth / rife49.pth), 417 (rife417.pth) or 426 (rife426.pth: five
 * blocks, scale list [16,8,4,2,1]/scale_factor, rife/__init__.py:156-158; CKPT_NAME_VER_DICT rife/__init__.py:10-14;
 * state_dict order = blocks 0..3 then encode.0.weight, encode.0.bias, encode.1.weight, encode.1.bias).  The
 * vfi_rife46_forward / _interpolate_host entry points below run whichever arch was loaded. */
int vfi_rife_load(vfi_ctx* ctx, int arch, const float* const* tensors, const int64_t* numel, int n_tensors,
                  int operand_type);

/* Replaces: the body of the hot loop of RIFE_VFI.vfi - rife/__init__.py:185-207 - i.e.
 *   IFNet.forward(frame[f0[i]], frame[f1[i]], t[i], scale_list=[8,4,2,1]/scale_factor).clamp(0,1)
 * for n_tasks (pair, timestep) tasks.  DEVICE pointers:
 *   frames : [n_frames, H, W, C] float32 NHWC, C >= 3 (only the first 3 channels are read, vfi_utils.py:139)
 *   out    : [n_tasks, H, W, 3] float32 NHWC
 * scale_factor: the node's widget (rife/__init__.py:49, :156-160), one of 0.25, 0.5, 1, 2, 4 (with 2 / 4 the last one / two
 * blocks run on an up-scaled input).
 * Asynchronous on `stream`. */
int vfi_rife46_forward(vfi_ctx* ctx, const float* frames, int n_frames, int H, int W, int C, const int32_t* f0,
                       const int32_t* f1, const float* t, int n_tasks, float scale_factor, float* out, void* stream);

/* Replaces: the whole per-batch loop incl. `.to(device)` / `.cpu()` - rife/__init__.py:185-222 - with a
 * pipelined H2D / compute / D2H schedule.  HOST pointers (pinned memory gives full PCIe rate; pageable works):
 *   frames : [n_frames, H, W, C] float32;  out : frames of [H, W, 3] float32.
 * Task i is written to out + out_slot[i]*H*W*3 (out_slot == NULL: slot i), so the caller can have the
 * interpolated frames land directly between the pass-through frames of the node's output tensor
 * (rife/__init__.py:225-238) without a second host copy.
 * Only frames in [frame_lo, frame_hi) are uploaded (the shard of this rank); tasks must reference only those.
 * frame_slot (NULL or [n_frames]): source frame f in [frame_lo, frame_hi) with frame_slot[f] >= 0 is also copied unchanged
 * (first 3 channels) to out + frame_slot[f]*H*W*3 - the pass-through frames of rife/__init__.py:227-231 - by the library's
 * copy threads; with a page-locked `out` that copy doubles as the staging copy of the upload.
 * Pageable `frames` / `out` go through pinned staging rings (VFI_STAGE_MB, VFI_COPY_THREADS); the prepared-frame window
 * on the device is a ring of ~2 x batch + 1 frames whatever the clip length.
 * Synchronous: returns when `out` is complete. */
int vfi_rife46_interpolate_host(vfi_ctx* ctx, const float* frames, int n_frames, int H, int W, int C, int frame_lo,
                                int frame_hi, const int32_t* f0, const int32_t* f1, const float* t,
                                const int32_t* out_slot, const int32_t* frame_slot, int n_tasks, float scale_factor,
                                float* out);

/* Host utility for the node's output assembly (rife/__init__.py:225-238: every source frame is passed through between
 * the interpolated ones): frame i (first 3 of C channels) -> out + slot[i]*H*W*3 for every i with slot[i] >= 0, split over
 * `threads` host threads.  HOST pointers, any host memory; no GPU involved.  Runs beside vfi_rife46_interpolate_host. */
int vfi_host_copy_frames(const float* frames, int n_frames, int H, int W, int C, const int32_t* slot, float* out, int threads);

/* Primitive: backward bilinear warp == rife_arch.warp (rife_arch.py:31-70) ==
 * grid_sample(bilinear, padding_mode="border", align_corners=True) on a pixel-unit flow.  DEVICE pointers, NHWC:
 * img [B,H,W,C] float32, flow [B,H,W,2] float32 (x, y displacement in pixels), out [B,H,W,C]. */
int vfi_warp_bilinear_border(vfi_ctx* ctx, const float* img, const float* flow, float* out, int B, int H, int W, int C,
                             void* stream);

/* Op-level surface of vfi_models/ops (the names the reference's models import, vfi_models/ops/__init__.py:19-21).
 * DEVICE pointers, contiguous NCHW float32 exactly like the reference's cupy launches (cupy_ops/softsplat.py:206-224).
 *   vfi_softsplat_sum : softsplat_out (cupy_ops/softsplat.py:140-192): out[N,C,H,W] (zeroed here) += forward splat of in
 *                       along flow [N,2,H,W]; the avg/linear/soft modes are host-side arithmetic around it (:382-435)
 *   vfi_costvol_l1    : costvol_out (cupy_ops/costvol.py:4-43): out[N,81,H,W] = mean_c |one - two(+-4 shifted)|
 *   vfi_corr_dot      : kernel_Correlation_updateOutput (cupy_ops/correlation.py:31-99): out[N,81,H,W], zero padded
 *   vfi_sepconv       : sepconv_out (cupy_ops/sepconv.py:86-117): in [N,C,H+Kv-1,W+Kh-1], ver [N,Kv,H,W], hor [N,Kh,H,W] */
int vfi_softsplat_sum(vfi_ctx* ctx, const float* in, const float* flow, float* out, int N, int C, int H, int W,
                      void* stream);
/* Fused form of the wrapper modes of softsplat() (cupy_ops/softsplat.py:382-435): mode 0 avg, 1 linear, 2 soft (weight 1,
 * metric, exp(metric) per source pixel), eps 0 addeps (default) / 1 zeroeps / 2 clipeps; `norm` is a caller-provided
 * [N,1,H,W] scratch plane (the splatted weights); out [N,C,H,W] = splat(in * weight) / f(norm).  metric may be NULL for avg. */
int vfi_softsplat_weighted(vfi_ctx* ctx, const float* in, const float* flow, const float* metric, int mode, int eps, float* out,
                           float* norm, int N, int C, int H, int W, void* stream);
int vfi_costvol_l1(vfi_ctx* ctx, const float* one, const float* two, float* out, int N, int C, int H, int W,
                   void* stream);
int vfi_corr_dot(vfi_ctx* ctx, const float* first, const float* second, float* out, int N, int C, int H, int W,
                 void* stream);
int vfi_sepconv(vfi_ctx* ctx, const float* in, const float* ver, const float* hor, float* out, int N, int C, int H,
                int W, int Kv, int Kh, void* stream);
/*   vfi_adacof        : kernel_AdaCoF_updateOutput (cupy_ops/adacof.py:5-62, wrapper :259-330): in [N,C,Hin,Win], weight /
 *                       offset_i / offset_j [N,F*F,Ho,Wo] with Hin = Ho + (F-1)*dilation, out [N,C,Ho,Wo]
 *   vfi_edt_pass      : kernel_dt (cupy_ops/batch_edt.py:9-41): one row pass of the separable squared distance transform,
 *                       data / out [bs,h,w]; batch_edt (:46-117) runs it twice around a transpose */
int vfi_adacof(vfi_ctx* ctx, const float* in, const float* weight, const float* offset_i, const float* offset_j, float* out,
               int N, int C, int Hin, int Win, int F, int dilation, int Ho, int Wo, void* stream);
int vfi_edt_pass(vfi_ctx* ctx, const float* data, float* out, int bs, int h, int w, float diam2, void* stream);

/* FILM (film_net) - SURVEY.md section 8 row a10 --------------------------------------------------------- */
#define VFI_FILM_NUM_TENSORS 82      /* film_arch.Interpolator().state_dict() (film_arch.py:377-393) */
/* Replaces: torch.jit.load(film_net_fp32.pt) - film/__init__.py:74.  `tensors[i]` are HOST float32 arrays in the
 * order of Interpolator.state_dict() (extract.extract_sublevels.convs.{0..3}.{0,1}.0.{weight,bias}, predict_flow.
 * _predictor._convs.{0..3}.0 / .4, predict_flow._predictors.{0,1,2}._convs..., fuse.output_conv, fuse.convs.{0..3}.
 * {0, 1.0, 2.0}); sizes are checked.  Weights are repacked to the streamed tensor-core operand layout. */
int vfi_film_load(vfi_ctx* ctx, const float* const* tensors, const int64_t* numel, int n_tensors, int operand_type);
/* Replaces: `model(x0, x1, dt)` in film/__init__.py:35-38 (Interpolator.forward, film_arch.py:458-459; the network
 * always predicts the midpoint, `dt` is not an input) for n_pairs independent pairs, optionally followed by the
 * node's clamp(0, 1) (:38).  DEVICE pointers: frames [n_frames, H, W, C] float32 NHWC (C >= 3, first three channels
 * read, vfi_utils.py:139), out [n_pairs, H, W, 3] float32 NHWC; f0 / f1: HOST index arrays.  H, W >= 64 (seven
 * pyramid levels), any other size as in the reference.  Asynchronous on `stream`. */
int vfi_film_forward(vfi_ctx* ctx, const float* frames, int n_frames, int H, int W, int C, const int32_t* f0,
                     const int32_t* f1, int n_pairs, int clamp01, float* out, void* stream);
/* Test / profiling hooks: route every FILM conv through the CUDA-core checker (1) or the wgmma kernel (0); run one
 * conv layer (group 0 = extract: layer 2*j + {0,1}; 1 = flow estimators: 4*predictor + conv; 2 = fusion: 3*k + conv)
 * on caller tensors (16-bit NHWC channel slices: pointer + pixel pitch in elements); static plan of a layer; tensor-core
 * MACs (unpadded channels) of the last forward. */
int vfi_film_debug_set_ref(vfi_ctx* ctx, int use_ref);
int vfi_film_debug_conv(vfi_ctx* ctx, int group, int layer, const void* src0, int pitch0, const void* src1, int pitch1,
                        void* out, int out_pitch, int B, int H, int W, int impl, void* stream);
int vfi_film_layer_plan(vfi_ctx* ctx, int group, int layer, int* c0, int* c1, int* n_total, int* ksize, int* n_cta,
                        int* nsplit, int* mt, int* a_slots, int* b_slots, int* smem_bytes);
int64_t vfi_film_last_macs(const vfi_ctx* ctx);
/* Test hooks.  vfi_film_debug_state copies the flow v[dir][level] of the last forward (dir 0 forward, 1 backward; level
 * 0..6, [batch, H_l, W_l, 2] float32) into a caller DEVICE buffer and synchronises; `out` NULL only returns H_l, W_l.
 * vfi_film_debug_elem runs one kernel of film_elem.cu on caller DEVICE tensors (16-bit slices: pointer + pixel pitch in
 * elements) with the loaded operand type and weights; asynchronous on `stream`.  kernel:
 *   0 gather_rgb  in0 frames [*, H, W, C] float32 -> out [B, H, W, 3]; frame_idx: HOST, B (<= 32) source frames
 *   1 pool_rgb    in0 [B, H, W, 3] -> out [B, H/2, W/2, 3] float32
 *   2 conv_rgb    in0 [B, H, W, 3] float32 -> out 64 channels (extract.convs.0.0 + LeakyReLU)
 *   3 pool16      in0 C channels at H x W -> out at H/2 x W/2
 *   4 flow_up     in0 flow [B, h, w, 2] -> out 2 * bilinear resize [B, H, W, 2] float32
 *   5 warp16      in0 C channels, in1 flow [B, H, W, 2] float32 scaled by fscale -> out C channels
 *   6 misc64      in0 / in1 images [B, H, W, 3], in2 backward / in3 forward flow -> out 64 channels
 *   7 nearest16   in0 [B, h, w, C] -> out [B, H, W, C] (both packed)
 *   8 flow_head   in0 C = nf/2 channels of predictor `predictor` (0..3), in1 up-sampled flow or NULL -> out flow float32
 *   9 out_rgb     in0 64 channels -> out [B, H, W, 3] float32, clamped to [0, 1] if clamp01
 * A launch the kernel's launcher refuses returns VFI_E_INVALID and names the reason. */
int vfi_film_debug_state(vfi_ctx* ctx, int dir, int level, float* out, int batch, int* H, int* W);
int vfi_film_debug_elem(vfi_ctx* ctx, int kernel, const void* in0, int in_pitch, const void* in1, const void* in2,
                        const void* in3, const int32_t* frame_idx, void* out, int out_pitch, int C, int B, int H, int W,
                        int h, int w, float fscale, int clamp01, int predictor, void* stream);
/* Host-only: vfi_film_load's weight packer on caller data (layout 0 = reference channel order padded to 64; layout 1 = a
 * fusion level's [wfeat0 C | wfeat1 C | misc 64] + nf decoder channels); `out` receives the packed 16-bit operand:
 * [split][k-block][tap][n_cta][64 ch, 16-byte chunks XOR (row & 7)]. */
int vfi_film_debug_pack_host(int layout, int C, int nf, int ksize, int n_total, int operand_type, const float* w,
                             int cout, int cin, uint16_t* out, int64_t out_cap, int* c0, int* c1, int* n_cta,
                             int* nsplit);

/* Sepconv (`Sepconv VFI` node) - SURVEY.md section 8 row a12 -------------------------------------------- */
#define VFI_SEPCONV_NUM_TENSORS 88   /* sepconv_enhanced.Network().state_dict() (sepconv_enhanced.py:536-598) */
/* Replaces: Network().load_state_dict(torch.load(path)) - sepconv/__init__.py:42-45.  HOST float32 arrays in
 * state_dict order (netInput, netEncode.0.netVer.{1..4}, netDecode.0.netHor.{0..3}, netDecode.0.netVer.{1..3}, netVerone,
 * netVertwo, netHorone, netHortwo); sizes are checked. */
int vfi_sepconv_load(vfi_ctx* ctx, const float* const* tensors, const int64_t* numel, int n_tensors, int operand_type);
/* Replaces: `model(frame_0, frame_1)` = Network.forward (sepconv_enhanced.py:605-706) for n_pairs independent pairs.
 * DEVICE pointers: frames [n_frames, H, W, C >= 3] float32 NHWC, out [n_pairs, H, W, 3] float32 NHWC (not clamped, like
 * the reference); f0 / f1: HOST index arrays.  Any H, W >= 2.  Asynchronous on `stream`. */
int vfi_sepconv_forward(vfi_ctx* ctx, const float* frames, int n_frames, int H, int W, int C, const int32_t* f0,
                        const int32_t* f1, int n_pairs, float* out, void* stream);
/* Test hooks: every conv through the CUDA-core checker (1) / the wgmma kernel (0); the host-only weight packer of
 * vfi_sepconv_load (a 3x3 conv packed as a stride-1 layer, or as the 2x2 conv over the space-to-depth input that runs
 * its stride-2 form). */
int vfi_sepconv_debug_set_ref(vfi_ctx* ctx, int use_ref);
/* Test hooks.  vfi_sepconv_debug_state copies a tensor of the last forward into a caller DEVICE buffer and synchronises;
 * `shape` (4 ints) receives its shape; `out` NULL only returns the shape.
 *   what 0: coefficient plane `index` (0 Verone, 1 Vertwo, 2 Horone, 3 Hortwo), [batch, 51, He, We] float32
 *   what 1: pyramid row `index` (1..4) after decoding, [batch, h_r, w_r, C_r] 16-bit
 *   what 2: per-pair statistics (sum, sum of squares of the padded pair), [batch, 2] double; index 0
 * vfi_sepconv_debug_elem runs one kernel of sepconv_elem.cu on caller DEVICE tensors with the loaded operand type;
 * asynchronous on `stream`.  He = H + (H & 1), We = W + (W & 1); 16-bit tensors are packed NHWC.  kernel:
 *   0 stats         in0 frames [n_frames, H, W, C] float32, pairs (f0[i], f1[i]) (HOST) -> out [B, 2] double
 *   1 input_conv    in0 frames, in1 stats [B, 2] double -> out [B, He/2, We/2, 128] (netInput + PReLU, space-to-depth)
 *   2 prelu_s2d16   in0 [B, H, W, C] -> out [B, ceil(H/2), ceil(W/2), 4 C], PReLU `slope`
 *   3 prelu16       in0 [B, H, W, C] -> out [B, H, W, C], PReLU `slope`
 *   4 prelu_up2_16  in0 [B, h, w, C] -> out [B, H, W, C] (H <= 2h, W <= 2w), PReLU `slope` then bilinear x2
 *   5 add_crop16    out [B, H, W, C] += in0 [B, h, w, C][:, :H, :W] (h >= H, w >= W)
 *   6 coeff_nchw    in0 [B, H, W, 64] -> out [B, 51, H, W] float32
 *   7 pad_input     in0 frames, frame f0[i] (which 0) or f1[i] (which 1) -> out [B, 4, He + 50, We + 50] float32
 *   8 finish        in0 / in1 [B, 4, He, We] float32 -> out [B, H, W, 3] float32
 * Arguments are checked before anything runs; a refused call returns VFI_E_INVALID, names the reason and writes nothing. */
int vfi_sepconv_debug_state(vfi_ctx* ctx, int what, int index, void* out, int batch, int* shape);
int vfi_sepconv_debug_elem(vfi_ctx* ctx, int kernel, const void* in0, const void* in1, const int32_t* f0, const int32_t* f1,
                           int n_frames, void* out, int C, int B, int H, int W, int h, int w, float slope, int which,
                           void* stream);
int vfi_sepconv_debug_pack_host(int stride2, int cin, int cout, int n_total, int operand_type, const float* w, uint16_t* out,
                                int64_t out_cap, int* c0, int* n_cta, int* nsplit);

/* FLAVR (`FLAVR VFI` node: UNet_3D_3D "unet_18", 4 input frames) ---------------------------------------- */
#define VFI_FLAVR_NUM_TENSORS 59       /* UNet_3D_3D.state_dict() without encoder conv biases (FLAVR_2x.pth) */
#define VFI_FLAVR_NUM_TENSORS_BIAS 76  /* with them (FLAVR_4x.pth, FLAVR_8x.pth: resnet_3D.useBias) */
#define VFI_FLAVR_MAX_WINDOWS 8
/* Replaces: build_flavr(path) - flavr/__init__.py:14-23.  HOST float32 arrays in UNet_3D_3D.state_dict() order (engine.py
 * flavr_state_dict_names); the tensor count tells whether the encoder convs carry a bias, the size of outconv.1.weight
 * the number of outputs (3 x n_outputs channels; only output 0 is used).  Sizes are checked. */
int vfi_flavr_load(vfi_ctx* ctx, const float* const* tensors, const int64_t* numel, int n_tensors, int operand_type);
/* Replaces: `model([f0, f1, f2, f3])[0]` on the InputPadder(16)-padded frames + padder.unpad (flavr/__init__.py:67-84,
 * :110) for n_windows windows: window k reads frames first_frame[k] .. first_frame[k] + 3.  DEVICE pointers: frames
 * [n_frames, H, W, C] float32 NHWC (C >= 3, first three channels read), out [n_windows, H, W, 3] float32 NHWC (not
 * clamped, like the reference); first_frame: HOST array.  Asynchronous on `stream`. */
int vfi_flavr_forward(vfi_ctx* ctx, const float* frames, int n_frames, int H, int W, int C, const int32_t* first_frame,
                      int n_windows, float* out, void* stream);
/* Test hooks: every conv through the CUDA-core checker (1) / the wgmma kernel (0); run one conv layer (id: encoder
 * 10 * layer + 3 * block + {0 conv1, 1 conv2, 2 downsample}; decoder 40 + 4 * d + phase; 60 feature_fuse) on caller
 * tensors [n_windows * T_in][H][W][pitch] 16-bit -> [n_windows * T_out][H][W][out_pitch]; its plan as
 * {c0, c1, n_total, ksize, kt, pad_t, T_in, T_out, pad_y, pad_x, n_cta, nsplit, a_slots, b_slots, smem_bytes, ext};
 * the loaded checkpoint's n_outputs and encoder-bias flag. */
int vfi_flavr_debug_set_ref(vfi_ctx* ctx, int use_ref);
int vfi_flavr_debug_conv(vfi_ctx* ctx, int layer, const void* src0, int pitch0, const void* src1, int pitch1, void* out,
                         int out_pitch, int n_windows, int H, int W, int impl, void* stream);
int vfi_flavr_layer_plan(vfi_ctx* ctx, int layer, int32_t* info, int cap);
int vfi_flavr_info(vfi_ctx* ctx, int* n_outputs, int* enc_bias);

/* IFRNet (`IFRNet VFI` node: IRFNet_S / IRFNet_L) ---------------------------------------------------------- */
#define VFI_IFRNET_NUM_TENSORS 104
/* Replaces: IRFNet_S() / IRFNet_L() + load_state_dict (ifrnet/__init__.py:44-45).  HOST float32 arrays in
 * state_dict() order (engine.py ifrnet_state_dict_spec); the variant is read from the first tensor's size, and every
 * tensor's size is checked against it. */
int vfi_ifrnet_load(vfi_ctx* ctx, const float* const* tensors, const int64_t* numel, int n_tensors, int operand_type);
/* Replaces: `model(img0, img1, scale_factor=t, timestep=embt)` for one pair (IRFNet_S.forward).  DEVICE pointers: img0,
 * img1 and out are float32 [3][H][W] planes (NCHW, batch 1); out is clamped to [0, 1].  t is the resize factor of the
 * encoder input, embt the value of decoder 4's time plane.  Sizes follow the reference's arithmetic; a t that gives an
 * empty encoder input or an output smaller than the frame is refused before any launch.  Asynchronous on `stream`. */
int vfi_ifrnet_forward(vfi_ctx* ctx, const float* img0, const float* img1, int H, int W, double t, double embt, float* out,
                       void* stream);
/* The sizes vfi_ifrnet_forward would use (no context): {Hp, Wp, encoder input h, w, levels 1..4 h, w, decoder 3..1 grids
 * h, w, decoder 1 output h, w, final resize h, w} (22 values), or the error it would return. */
int vfi_ifrnet_geometry(int H, int W, double t, int32_t* info, int cap);
/* Test hooks: every conv through the CUDA-core checker (1) / the wgmma kernel (0); run one conv layer (id: encoder
 * 0..6 = pyramid1.1, pyramid2.0 (stride 2, space-to-depth input), pyramid2.1, ..; decoder k = 0 (decoder4) .. 3:
 * 10 + 10 k + {0 convblock.0, 1..5 ResBlock conv1..conv5, 6..9 ConvT phase py * 2 + px}); its plan
 * {c0, c1, n_total, ksize, pad_y, pad_x, n_cta, nsplit, a_slots, b_slots, smem_bytes, n_f32}; the loaded variant
 * (0: IFRNet-S, 1: IFRNet-L). */
int vfi_ifrnet_debug_set_ref(vfi_ctx* ctx, int use_ref);
int vfi_ifrnet_debug_conv(vfi_ctx* ctx, int layer, const void* src0, int pitch0, const void* src1, int pitch1, void* out,
                          int out_pitch, const void* res, float* out_f32, int f32_pitch, int n_images, int H, int W,
                          int impl, void* stream);
int vfi_ifrnet_layer_plan(vfi_ctx* ctx, int layer, int32_t* info, int cap);
int vfi_ifrnet_info(vfi_ctx* ctx, int* variant);

/* CAIN (`CAIN VFI` node: CAIN(depth=3)) ---------------------------------------------------------------------- */
#define VFI_CAIN_NUM_TENSORS 494
/* Replaces: CAIN(depth=3).load_state_dict(sd) with the checkpoint's "module." prefix stripped (cain/__init__.py:
 * 42-48).  HOST float32 arrays in state_dict() order (engine.py cain_state_dict_spec); every tensor's size is checked and
 * a refusal names the tensor. */
int vfi_cain_load(vfi_ctx* ctx, const float* const* tensors, const int64_t* numel, int n_tensors, int operand_type);
/* Replaces: `model(img0, img1)[0]` for one pair (CAIN.forward, cain_arch.py).  DEVICE pointers: img0, img1 and out are
 * float32 [3][H][W] planes (NCHW, batch 1); out is not clamped.  A frame the reference's ReflectionPad2d cannot pad
 * (padding on a side not smaller than the axis) is refused before any launch.  Asynchronous on `stream`. */
int vfi_cain_forward(vfi_ctx* ctx, const float* img0, const float* img1, int H, int W, float* out, void* stream);
/* The sizes vfi_cain_forward would use (no context): {Hp, Wp, trunk grid h, w, padding top, left} (6 values), or the
 * error it would return. */
int vfi_cain_geometry(int H, int W, int32_t* info, int cap);
/* Test hooks: every conv through the CUDA-core checker (1) / the wgmma kernel (0); run one conv layer (id: 0 headConv,
 * 1 + 25 g + 2 r + {0 conv1, 1 conv2} of RCAB r in group g, 1 + 25 g + 24 the group's tail conv, 126 tailConv) on
 * 16-bit NHWC slices; its plan {c0, c1, n_total, ksize, act, ext, n_cta, nsplit, a_slots, b_slots, smem_bytes}.
 * vfi_cain_debug_elem runs one element-wise stage for an H x W frame on DEVICE tensors of the bordered grid
 * ((h + 2) x (w + 2) cells of 192 16-bit channels, h x w from vfi_cain_geometry): kernel 0 prep (img0, img1 -> out of
 * 384 channels), 1 reflected border of out (in place), 2 zero border of out and res added to its interior, 3 channel
 * attention of RCAB `rcab` (0..59): out = x * gate(mean of x's interior) + res on every cell, 4 final (x, with the
 * means of img0 and img1 -> out float32 [3][H][W]).  Asynchronous on `stream`. */
int vfi_cain_debug_set_ref(vfi_ctx* ctx, int use_ref);
int vfi_cain_debug_conv(vfi_ctx* ctx, int layer, const void* src0, int pitch0, const void* src1, int pitch1, void* out,
                        int out_pitch, const void* res, int n_images, int H, int W, int impl, void* stream);
int vfi_cain_layer_plan(vfi_ctx* ctx, int layer, int32_t* info, int cap);
int vfi_cain_debug_elem(vfi_ctx* ctx, int kernel, const float* img0, const float* img1, int H, int W, const void* x,
                        const void* res, void* out, int rcab, void* stream);

/* IFUnet (`IFUnet VFI` node: IFUNetModel, IFUNet.pth) ------------------------------------------------------- */
#define VFI_IFUNET_NUM_TENSORS 608
/* Replaces: IFUNetModel().load_state_dict(torch.load(path)) (ifunet/__init__.py).  HOST float32 arrays in state_dict()
 * order (engine.py ifunet_state_dict_spec; the num_batches_tracked scalars and the unused refinenet.degrad tensors
 * included); every tensor's size is checked and a refusal names the tensor.  Eval-mode BatchNorm is folded at load. */
int vfi_ifunet_load(vfi_ctx* ctx, const float* const* tensors, const int64_t* numel, int n_tensors, int operand_type);
/* Replaces: `model(img0, img1, timestep=t, scale=scale, ensemble=ensemble)` for one pair (IFUNetModel.forward).
 * DEVICE pointers: img0, img1 and out are float32 [3][H][W] planes (NCHW, batch 1).  A scale at which the reference
 * raises (a UpConv input that does not double to its skip connection, or a level's flow that does not come back to the
 * padded size) and a workspace the device cannot hold are refused before any launch.  Asynchronous on `stream`. */
int vfi_ifunet_forward(vfi_ctx* ctx, const float* img0, const float* img1, int H, int W, double timestep, double scale,
                       int ensemble, float* out, void* stream);
/* The sizes vfi_ifunet_forward would use (no context): {Hp, Wp, then h, w of the flow net's input and of its five
 * stride-2 levels} (14 values), or the error it would return. */
int vfi_ifunet_geometry(int H, int W, double scale, int32_t* info, int cap);
/* Test hooks: every conv through the CUDA-core checker (1) / the wgmma kernel (0); run one conv layer (ids in
 * csrc/ifunet.cu) on 16-bit NHWC slices, with its residual and fp32 columns; its plan {c0, c1, n_total, ksize, act,
 * ext, n_f32, pad_before, pad_before_x, n_cta, nsplit, a_slots, b_slots, smem_bytes}.  vfi_ifunet_debug_elem runs one
 * element-wise stage on DEVICE tensors: kernel 0 the level-0 input of `index` (1 or 2) images of an H x W pair at
 * `scale` / `timestep` (img0, img1 -> out, the 128-channel space-to-depth copy), 1 CBAM `index` (0..3: FeatureNet conv2
 * .. conv5, 4: deconv5) in place on out [H][W][C], 2 the convex upsampling of IFBlock `index` (x: flow fp32 [H][W][4],
 * y: mask logits [H][W][9 L L] 16-bit -> out fp32 [L H][L W][4]), 3 the warps of an H x W pair by x = flow fp32
 * [Hp][Wp][4] -> out fp32 [2][3][Hp][Wp].  Asynchronous on `stream`. */
int vfi_ifunet_debug_set_ref(vfi_ctx* ctx, int use_ref);
int vfi_ifunet_debug_conv(vfi_ctx* ctx, int layer, const void* src0, int pitch0, const void* src1, int pitch1, void* out,
                          int out_pitch, const void* res, float* out_f32, int f32_pitch, int B, int H, int W, int impl,
                          void* stream);
int vfi_ifunet_layer_plan(vfi_ctx* ctx, int layer, int32_t* info, int cap);
int vfi_ifunet_debug_elem(vfi_ctx* ctx, int kernel, const float* img0, const float* img1, int H, int W, double timestep,
                          double scale, const void* x, const void* y, void* out, int index, void* stream);

/* Test / profiling hooks (used by tests/ and bench.py only) --------------------------------------------- */
/* Run ONE convolution layer of block `block` (0..3; arch 4.26: 0..4): layer 0 = conv0.0, 1 = conv0.1, 2..9 = ResConv
 * 0..7, 10 = lastconv (flow + mask), 11 = arch 4.26 blocks 0..3: the 8 feature channels of lastconv, written as
 * [B, 4H, 4W, 8] 16-bit.  `in`/`out` are device tensors in the kernel-native layouts documented in DESIGN.md
 * (16-bit NHWC; layers 0/1 read space-to-depth inputs; layer 10 writes float4 flow + float mask planes).
 * impl 0 = wgmma kernel as planned, 1 = CUDA-core checker with the same packed weights, 2 = wgmma kernel with the
 * grid cells on the MMA's M even where the plan runs the layer channel-major (see vfi_rife46_layer_plan). */
int vfi_rife46_debug_layer(vfi_ctx* ctx, int block, int layer, const void* in, void* out, void* out_mask, int B, int H,
                           int W, int impl, void* stream);
/* Copies the full-resolution flow (float4 [batch,Hp,Wp]) and mask (float [batch,Hp,Wp]) of the LAST internal
 * pass into caller-provided DEVICE buffers (either may be NULL to only query Hp/Wp); synchronises. */
int vfi_rife46_debug_state(vfi_ctx* ctx, float* flow4_out, float* mask_out, int batch, int* Hp, int* Wp);
/* Static plan of a layer for (block, layer): shared-memory stages, CTA output channels, splits, smem bytes, MACs per
 * grid cell, cmajor = 1 when the layer runs channel-major (output channels on the MMA's M, 128 cells on N) and
 * wstream = 1 when its weights stream through shared memory instead of staying resident (any pointer may be NULL). */
int vfi_rife46_layer_plan(vfi_ctx* ctx, int block, int layer, int* stages, int* n_cta, int* nsplit, int* smem_bytes,
                          int64_t* macs_per_cell, int* cmajor, int* wstream);
/* conv0.0 and conv0.1 of arch 4.6's 64-channel block (block 3) run as one launch whenever that block runs at full
 * resolution (scale 1): conv0.0's output stays in shared memory (DESIGN.md section 4.1).  vfi_rife46_debug_conv0_fused
 * runs that launch alone over `in` (the block input, 16-bit [B, H, W, 64] space-to-depth cells) into `out` (16-bit
 * [B, H/2, W/2, 64]); VFI_E_INVALID for a block whose layers it cannot run.  vfi_rife46_debug_unfused_conv0(ctx, 1) makes
 * the forward schedule run that block's conv0.0 and conv0.1 as two launches instead (0: back to one), the tests'
 * reference.  vfi_rife46_conv0_plan: info[0..4] = {1 when the block's pair can run fused (at scale 1), its x window
 * stages, shared-memory bytes, registers per thread, local (spill) bytes per thread}, all 0 otherwise (at most cap). */
int vfi_rife46_debug_conv0_fused(vfi_ctx* ctx, int block, const void* in, void* out, int B, int H, int W, void* stream);
int vfi_rife46_debug_unfused_conv0(vfi_ctx* ctx, int unfused);
int vfi_rife46_conv0_plan(vfi_ctx* ctx, int block, int32_t* info, int cap);
int vfi_sync(vfi_ctx* ctx);
/* Run ONE streamconv layer (csrc/streamconv.cu, the conv kernel of FILM, Sepconv, FLAVR, IFRNet and CAIN) from a plain
 * description, without a model: spec = {ksize, c0, c1, n_total, act, ext, n_f32, pad_before, pad_before_x, kt, pad_t,
 * T_in, T_out} (the fields of the layer; n_spec = 13), slope = the ext 1 PReLU slope.  HOST fp32: w [n_total][kt]
 * [ksize * ksize][c0 + c1], shift [n_total], slopes [n_total] (ext 2; may be NULL otherwise); they are packed by the
 * product packer into temporary device buffers.  DEVICE: the 16-bit NHWC source / output / residual slices (pointer +
 * pixel pitch in elements; B samples of T_in / T_out planes) and the fp32 slice of the first n_f32 columns.
 * num_sms <= 0: the device's SM count (a smaller value makes every CTA walk more passes).  impl 0 = wgmma kernel,
 * 1 = CUDA-core checker.  Synchronises `stream`; returns the launch's or the run's error. */
int vfi_streamconv_debug_conv(const int32_t* spec, int n_spec, float slope, int operand_type, const float* w,
                              const float* shift, const float* slopes, const void* src0, int pitch0, const void* src1,
                              int pitch1, void* out, int out_pitch, const void* res, float* out_f32, int f32_pitch, int B,
                              int H, int W, int num_sms, int impl, void* stream);
/* The plan of such a layer: {n_cta, nsplit, a_slots, b_slots, smem_bytes, halo_y0, halo_x0}, or VFI_E_INVALID when
 * streamconv cannot run it.  No GPU needed. */
int vfi_streamconv_plan(const int32_t* spec, int n_spec, int32_t* info, int cap);

/* Measurement hook (bench.py's roofline lines): while enabled, every internal pass of the RIFE forward schedule records
 * CUDA events on its launching stream around each kernel group - id = 10 * block + {0 front (warps + resample + concat,
 * rife_arch.py:238-249, :703-704), 1 conv0.0, 2 conv0.1, 3 the eight ResConvs, 4 lastconv}, 90 = the final warp / blend /
 * crop kernel (rife_arch.py:713-732).  vfi_rife_profile_read synchronises and returns, per group id, the summed device
 * time in ms and the number of spans; at most `cap` groups.  No counterpart in the reference (it has no timing code). */
int vfi_rife_profile(vfi_ctx* ctx, int enable);
int vfi_rife_profile_read(vfi_ctx* ctx, int32_t* ids, float* total_ms, int32_t* count, int cap, int* n_groups);

/* ---------------------------------------------------------------------------------------------------------------------
 * GMFSS Fortuna (union) building blocks - csrc/gmops.cu; the schedule that strings them together is host code
 * (comfyui-frame-interpolation_b200/gmfss.py), mirroring vfi_models/gmfss_fortuna/GMFSS_Fortuna_union_arch.py :1726-1857.
 * They replace what that file runs through ATen / cuDNN / cuBLAS between its softsplat calls: F.conv2d / conv_transpose2d
 * with the nn.PReLU in front and the residual adds behind (:1420-1688, :165-312), F.instance_norm (:165-215), nn.Linear /
 * torch.matmul / softmax / LayerNorm / GELU of the swin transformer (:315-685) and of the flow propagation (:688-803),
 * split_feature / merge_splits with torch.roll (:366-436, :1059-1131), PositionEmbeddingSine (:1015-1056),
 * local_correlation_softmax (:846-913), upsample_flow (:1220-1260), grid_sample / F.interpolate (:955-991, :1375-1417),
 * MetricNet's input assembly with the forward-backward check (:994-1013, :1429-1455), F.pixel_shuffle, torch.cat / slicing.
 * DEVICE pointers, contiguous float32, NCHW tensors (tokens: [B, L, C]); `stream` is the caller's CUDA stream; 0 = OK.
 * Argument meaning is documented at each kernel in csrc/gmops.cu. */
int vfi_gm_conv2d(const float* in, const float* w, const float* bias, const float* res1, const float* res2, float* out, int N, int Cin, int H, int W, int Cout, int k, int stride, int pad, int in_ctot, int in_coff, int out_ctot, int out_coff, int has_pre, float pre_slope, int post, float post_slope, void* stream);
int vfi_gm_conv2d_packed(const float* in, const float* wt, const float* bias, const float* res1, const float* res2, float* out, int N, int Cin, int H, int W, int Cout, int CoutP, int k, int stride, int pad, int in_ctot, int in_coff, int out_ctot, int out_coff, int has_pre, float pre_slope, int post, float post_slope, void* stream);
int vfi_gm_transpose(const float* src, float* dst, int nb, int R, int C, void* stream);
int vfi_gm_convt4(const float* in, const float* w, const float* bias, float* out, int N, int Cin, int H, int W, int Cout, int has_pre, float pre_slope, void* stream);
int vfi_gm_instance_norm(const float* in, float* out, int planes, int HW, float eps, int relu, void* stream);
int vfi_gm_layer_norm(const float* x, const float* gamma, const float* beta, const float* src, float* out, int rows, int C, float eps, void* stream);
int vfi_gm_softmax_rows(float* x, int rows, int L, void* stream);
int vfi_gm_gemm(int bt, const float* A, const float* B, const float* bias, const float* mask, float* C, int nb, int M, int N, int K, int lda, int ldb, int ldc, long long sA, long long sB, long long sC, float alpha, int nmask, int act, void* stream);
int vfi_gm_window(const float* src, float* dst, int B, int H, int W, int C, int k, int sh, int sw, int to_windows, void* stream);
int vfi_gm_nchw_tokens(const float* src, float* dst, int B, int C, int HW, int to_tokens, void* stream);
int vfi_gm_add_position(float* x, int B, int C, int H, int W, int k, void* stream);
int vfi_gm_local_match(const float* f0, const float* f1, float* flow, int B, int C, int H, int W, int R, void* stream);
int vfi_gm_local_prop(const float* q, const float* k, const float* flow, float* out, int B, int C, int H, int W, void* stream);
int vfi_gm_convex_up(const float* mask, const float* flow, float* up, int B, int H, int W, int f, void* stream);
int vfi_gm_warp_zeros(const float* in, const float* flow, float* out, int B, int C, int H, int W, void* stream);
int vfi_gm_resize(const float* in, float* out, int BC, int H, int W, int Ho, int Wo, int align, float mul, void* stream);
int vfi_gm_metric_input(const float* img0, const float* img1, const float* f01, const float* f10, float* out, int B, int H, int W, void* stream);
int vfi_gm_pixel_shuffle2(const float* in, float* out, int B, int C, int H, int W, void* stream);
int vfi_gm_axpby(const float* a, const float* b, float* out, long long n, float alpha, float beta, float gamma, int post, void* stream);
int vfi_gm_copy_slice(const float* src, float* dst, int B, int C, int Hs, int Ws, int Hd, int Wd, int s_ctot, int s_coff, int d_ctot, int d_coff, int src_nhwc, int dst_nhwc, const float* mean, const float* stdv, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VFI_B200_H */
