// tapconv: tap-list implicit-GEMM convolution on the Hopper tensor cores (wgmma / TMA / mbarrier), sm_90a only.
//
// Replaces, for the RIFE IFBlock (reference rife_arch.py:237-276), the cuDNN/ATen kernels behind
//   conv0.0 / conv0.1  Conv2d(3x3, stride 2)+LeakyReLU        rife_arch.py:96-107, :181-184
//   convblock          8 x ResConv  lrelu(conv3x3(x)*beta + x) rife_arch.py:20-28, :201-210
//   lastconv           ConvTranspose2d(c,24,4,2,1)+PixelShuffle rife_arch.py:215-218
//
// One CTA tile = 16 x 8 grid cells = 128 GEMM rows, two m64 wgmma row blocks (tile rows 0-7 and 8-15).  The input
// window of the tile (tile + halo, all input channels) is dropped ONCE into shared memory by TMA as rows of 64 channels
//      A[k-block][window pixel][64 ch = 128 B, SWIZZLE_128B]      (a 32-channel SWIZZLE_64B tail when cin % 64 = 32)
// i.e. the canonical K-major swizzled wgmma operand with "rows = pixels".  TMA zero-fills everything outside the
// image, which implements both the convolution padding and partial border tiles.  Every filter tap is then just a
// different descriptor START ADDRESS into the same window (whole-row shift (dy*halo_w + dx) * 128 B, with the
// 8-row-group stride SBO = halo_w * 128 B), a K=16 step a 32-byte shift inside the row: the tensor core applies the
// XOR swizzle on the absolute shared-memory address, exactly where TMA put the data.  So the 3x3 window is read from L2
// once (x1.41 halo), not 9x as with im2col.  Weights of the CTA's output-channel slice are resident in shared memory
// for the whole launch (one bulk copy, already in the swizzled operand layout).
//
// Warp roles (288 threads, 1 CTA/SM, persistent over tiles):
//   warpgroups 0, 1 : MMA + epilogue.  Warpgroup w takes the CTA's tiles w, w + 2, ... and keeps the whole tile's
//                     accumulators (2 x 64 rows x n_cta columns, fp32) in registers, so one warpgroup's epilogue
//                     (+shift (+residual) -> LeakyReLU -> 16-bit -> global stores; lastconv: the fp32 4x4 flow/mask
//                     sub-pixel patch) overlaps the other's MMAs.
//   warp 8          : one elected lane: weight bulk copy, then one 4-D TMA tensor copy per k-block and tile
#include <cstdlib>
#include <type_traits>

#include "ptx.cuh"
#include "vfi_internal.h"

namespace vfi {

namespace {

constexpr int kMaxStages = 6;   // window stages or ring slots
struct Ctrl {
  uint64_t w_full;
  uint64_t a_full[kMaxStages][2];  // [stage][consuming warpgroup]
  uint64_t a_empty[kMaxStages];
};
constexpr uint32_t kCtrlBytes = 256;
constexpr int kMmaGroups = 2, kTmaWarp = 8, kThreads = 128 * kMmaGroups + 32;
static_assert(sizeof(Ctrl) <= kCtrlBytes, "control block");

__device__ __forceinline__ size_t out_pixel_offset(const TapConvParams& p, int b, int gy, int gx) {
  // element offset of channel 0 of grid cell (b, gy, gx) in the output tensor
  if (p.out_s2d == 1) {
    // space-to-depth store: the consumer is a stride-2 conv that reads [B, H/2, W/2, 4*n_total]
    size_t cell = ((size_t)b * (p.H >> 1) + (gy >> 1)) * (p.W >> 1) + (gx >> 1);
    return cell * (size_t)(4 * p.n_total) + (size_t)(((gy & 1) * 2 + (gx & 1)) * p.n_total);
  }
  if (p.out_s2d == 2)  // patch form [B, 4H, 4W, 8]: element offset of sub-pixel (0, 0) of this cell's 4x4 patch
    return (((size_t)b * (4 * p.H) + 4 * gy) * (size_t)(4 * p.W) + 4 * gx) * 8;
  return (((size_t)b * p.H + gy) * p.W + gx) * (size_t)p.n_total;
}

#ifndef VFI_HOST_EMU  // (tests/host_emu runs the RIFE schedule on the CPU with the checker kernel; no wgmma there)
// Walks the tiles of one CTA (t = first, first + cps, ...) keeping (image, tile row, tile column) incrementally
// instead of two integer divisions per tile and role.
struct TileIter {
  int b, ty, tx, db, dy, dx, tiles_x, tiles_y;
  __device__ __forceinline__ TileIter(const TapConvParams& p, int first, int step) {
    tiles_x = p.tiles_x;
    tiles_y = p.tiles_y;
    const int per_img = tiles_x * tiles_y;
    b = first / per_img;
    int rem = first - b * per_img;
    ty = rem / tiles_x;
    tx = rem - ty * tiles_x;
    db = step / per_img;
    rem = step - db * per_img;
    dy = rem / tiles_x;
    dx = rem - dy * tiles_x;
  }
  __device__ __forceinline__ void next() {
    tx += dx;
    ty += dy;
    b += db;
    if (tx >= tiles_x) {
      tx -= tiles_x;
      ++ty;
    }
    if (ty >= tiles_y) {  // dy < tiles_y and the carry add at most tiles_y
      ty -= tiles_y;
      ++b;
    }
  }
};

// One window's MMAs for both 64-row halves of the tile: p.nruns runs of p.run_len consecutive K=16 steps (same tap,
// same k-block: both descriptors advance by 32 bytes per step).  a_base / b_base: start-address words (16-byte units,
// LBO = 1) of the window and of the weights of this k-block.
template <int N, typename T>
__device__ __forceinline__ void issue_window(const TapConvParams& p, float (&acc)[2][N / 2], uint32_t a_base,
                                             uint32_t b_base, uint32_t accumulate_first) {
#pragma unroll 1
  for (int r = 0; r < p.nruns; ++r) {
    const uint4 d = p.mma[r];
    const uint32_t half_off = 8u * (d.y & 0x3fffu);  // 8 tile rows further down the window = 8 SBO strides
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint64_t a64 = ((uint64_t)d.y << 32) | (uint64_t)(a_base + d.x + (uint32_t)h * half_off);
      uint64_t b64 = ((uint64_t)p.b_hi << 32) | (uint64_t)(b_base + d.z);
#pragma unroll 1
      for (int i = 0; i < p.run_len; ++i) {
        wgmma_ss<N, T>(acc[h], a64, b64, (r | i) ? 1u : accumulate_first);
        a64 += 2;
        b64 += 2;
      }
    }
  }
}

template <typename T, bool RING, bool LAST, int N>
__global__ void __launch_bounds__(kThreads, 1) tapconv_kernel(const __grid_constant__ TapConvParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  // Programmatic dependent launch (launch_tapconv sets the attribute): the next kernel in the stream may start its
  // CTAs as soon as every CTA of this grid has passed this point, i.e. while our last tiles are still running - they do
  // their prologue (barrier init, weight copy) on the SMs our first finishers free and then block in
  // griddepcontrol.wait until this grid has completed and flushed.  Both instructions are no-ops without the attribute.
  asm volatile("griddepcontrol.launch_dependents;");
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // CTA (split, first) takes the output-channel slice `split` of tiles first, first + cps, ...
  const int split = (int)blockIdx.x % p.nsplit;
  const int first = (int)blockIdx.x / p.nsplit;
  if (first >= p.ctas_per_split) return;  // whole CTA leaves together
  const int tstep = p.ctas_per_split;
  const int my_tiles = (p.ntiles - first + tstep - 1) / tstep;
  const int n0 = split * p.n_cta;  // first output channel of this CTA
  const int S = p.stages;
  const bool residual = !LAST && (p.epi_mode == EPI_RESCONV);

  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bar_w = smem_base + offsetof(Ctrl, w_full);
  const uint32_t bar_afull = smem_base + offsetof(Ctrl, a_full);
  const uint32_t bar_aempty = smem_base + offsetof(Ctrl, a_empty);
  const uint32_t a_smem = smem_base + p.off_a;
  const uint32_t w_smem = smem_base + p.off_w;
  const bool has_tail = (p.cin & 63) != 0;  // last k-block is 32 channels wide

  if (threadIdx.x == 0) {
    mbar_init(bar_w, 1);
    for (int s = 0; s < S; ++s) {
      mbar_init(bar_afull + 16 * s, 1);      // producer's arrive.expect_tx (+ TMA transaction bytes), per warpgroup
      mbar_init(bar_afull + 16 * s + 8, 1);
      mbar_init(bar_aempty + 8 * s, 4);      // the four warps of the consuming warpgroup
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == kTmaWarp) {
    // ======================================================= TMA producer (one thread feeds the whole pipeline)
    if (lane == 0) {
      mbar_arrive_expect_tx(bar_w, p.w_bytes);
      const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(p.w) + (size_t)split * p.w_bytes;
      for (uint32_t off = 0; off < p.w_bytes; off += 32768u)
        bulk_g2s(w_smem + off, wsrc + off, min(32768u, p.w_bytes - off), bar_w);
      // weights do not depend on the previous kernel; its output (our input tensor) does
      asm volatile("griddepcontrol.wait;" ::: "memory");
      TileIter it(p, first, tstep);
      uint32_t stage = 0, eph = 1;  // window stage / ring slot and the parity of its "empty" barrier
      for (int k = 0; k < my_tiles; ++k, it.next()) {
        const int gy0 = it.ty * kTileH + p.halo_y0, gx0 = it.tx * kTileW + p.halo_x0;
        if (RING) {
          for (int kb = 0; kb < p.nkb; ++kb) {
            const uint32_t full = bar_afull + 16 * stage + 8 * (k & 1);  // tile k goes to warpgroup k % 2
            mbar_wait(bar_aempty + 8 * stage, eph);
            mbar_arrive_expect_tx(full, p.tx_bytes);
            tma_load_4d(a_smem + stage * p.stage_bytes, &p.tm64, full, kb * 64, gx0, gy0, it.b);
            if (++stage == (uint32_t)S) {
              stage = 0;
              eph ^= 1u;
            }
          }
        } else {
          const uint32_t full = bar_afull + 16 * stage + 8 * (k & 1);
          mbar_wait(bar_aempty + 8 * stage, eph);
          mbar_arrive_expect_tx(full, p.tx_bytes);
          const uint32_t dst = a_smem + stage * p.stage_bytes;
          for (int kb = 0; kb < p.nkb; ++kb) {
            const bool tail = has_tail && (kb == p.nkb - 1);
            tma_load_4d(dst + p.kb_off[kb], tail ? &p.tm32 : &p.tm64, full, kb * 64, gx0, gy0, it.b);
          }
          if (++stage == (uint32_t)S) {
            stage = 0;
            eph ^= 1u;
          }
        }
      }
    }
    return;
  }

  // ========================================================= MMA + epilogue warpgroups
  // Warpgroup g consumes the stages of tiles g, g + 2, ... through its own "full" barrier of each stage: the fills a
  // warpgroup waits for on one barrier are its own, in order, so a parity wait never confuses an older phase with the
  // one it wants (a stage shared by both warpgroups would, with one or an odd number of stages).
  const int g = warp >> 2;
  const int wq = warp & 3;  // warp of the warpgroup: rows 16 wq .. 16 wq + 15 of each 64-row half
  // the previous kernel may still be reading the buffer we store to (ping-pong) and ResConv layers read the residual
  // from global memory: every storing / loading thread orders itself after the previous grid
  asm volatile("griddepcontrol.wait;" ::: "memory");
  mbar_wait(bar_w, 0);
  const uint32_t a_lo0 = (1u << 16) | (a_smem >> 4);  // LBO(=1) | start address, 16-byte units
  const uint32_t b_lo0 = (1u << 16) | (w_smem >> 4);
  const uint32_t per_tile = RING ? (uint32_t)p.nkb : 1u;  // stages / slots one tile consumes
  const uint32_t b_kb = (9u * (uint32_t)p.n_cta * 128u) >> 4;  // ring: weight bytes of one k-block, 16-byte units
  const uint32_t stage_units = p.stage_bytes >> 4;
  uint32_t stage = 0, ph_bits = 0;  // window stage / ring slot; bit s: parity of this warpgroup's next wait on stage s
  auto advance = [&](uint32_t n) {
    stage += n;
    while (stage >= (uint32_t)S) stage -= (uint32_t)S;
  };
  auto wait_full = [&]() {
    mbar_wait(bar_afull + 16 * stage + 8 * (uint32_t)g, (ph_bits >> stage) & 1u);
    ph_bits ^= 1u << stage;
  };
  advance((uint32_t)g * per_tile);
  const float slope = (p.epi_mode == EPI_BIAS) ? 1.f : 0.2f;  // max(a, slope * a): LeakyReLU(0.2), or no activation
  const int px = lane >> 2;             // tile column of this thread's accumulator rows
  const int c2 = 2 * (lane & 3);        // first of this thread's two columns in every 8-column block
  float acc[2][N / 2];

  TileIter it(p, first + g * tstep, kMmaGroups * tstep);
  for (int k = g; k < my_tiles; k += kMmaGroups, it.next()) {
    if (RING) {
      uint32_t prev = 0;
      for (int kb = 0; kb < p.nkb; ++kb) {
        wait_full();
        wgmma_fence();
        issue_window<N, T>(p, acc, a_lo0 + stage * stage_units, b_lo0 + (uint32_t)kb * b_kb, kb > 0 ? 1u : 0u);
        wgmma_commit();
        if (kb > 0) {  // the previous slot's MMAs have read it
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_aempty + 8 * prev);
        }
        prev = stage;
        advance(1u);
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_aempty + 8 * prev);
      advance(per_tile);  // the other warpgroup's tile
    } else {
      wait_full();
      wgmma_fence();
      issue_window<N, T>(p, acc, a_lo0 + stage * stage_units, b_lo0, 0u);
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_aempty + 8 * stage);  // window free once the MMAs have read it
      advance((uint32_t)kMmaGroups);
    }
    acc_fence(acc[0]);
    acc_fence(acc[1]);

    // ---- epilogue straight from the accumulator registers: d[h][4 j + 2 e + c] = tile row 8 h + 2 wq + e, column
    // 8 j + c2 + c
    const int b = it.b;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int gy = it.ty * kTileH + 8 * h + 2 * wq + e, gx = it.tx * kTileW + px;
        if (gy >= p.H || gx >= p.W) continue;
        if (LAST) {
          // column n = c5*16 + pos: component c5 (4 flow + mask) of sub-pixel pos = y4*4 + x4 of this cell's 4x4 patch
          const int Hs = p.H * 4, Ws = p.W * 4;
#pragma unroll
          for (int j = 0; j < N / 8; ++j) {
            const int n = n0 + 8 * j + c2;
            const float2 sh = __ldg(reinterpret_cast<const float2*>(p.shift + n));
            const int c5 = n >> 4, pos = n & 15;  // n even: n + 1 is the next sub-pixel of the same patch row
            const size_t o = ((size_t)b * Hs + (gy * 4 + (pos >> 2))) * Ws + gx * 4 + (pos & 3);
            const float v0 = acc[h][4 * j + 2 * e] + sh.x, v1 = acc[h][4 * j + 2 * e + 1] + sh.y;
            if (c5 < 4) {
              float* f = reinterpret_cast<float*>(p.out_flow + o);
              f[c5] = v0;
              f[4 + c5] = v1;
            } else {
              *reinterpret_cast<float2*>(p.out_mask + o) = make_float2(v0, v1);
            }
          }
        } else {
          const bool patch = (p.out_s2d == 2);
          T* orow = reinterpret_cast<T*>(p.out) + out_pixel_offset(p, b, gy, gx);
          const T* rrow = reinterpret_cast<const T*>(p.in) + (((size_t)b * p.H + gy) * p.W + gx) * (size_t)p.cin;
#pragma unroll
          for (int j = 0; j < N / 8; ++j) {
            const int n = n0 + 8 * j + c2;
            const float2 sh = __ldg(reinterpret_cast<const float2*>(p.shift + n));
            float a0 = acc[h][4 * j + 2 * e] + sh.x, a1 = acc[h][4 * j + 2 * e + 1] + sh.y;
            if (residual) {
              const float2 rf = Pack2<T>::unpack(__ldg(reinterpret_cast<const unsigned int*>(rrow + n)));
              a0 += rf.x;
              a1 += rf.y;
            }
            // patch form: columns n = sub-pixel (n >> 3) x channel (n & 7)
            const size_t off = patch ? ((size_t)((n >> 3) >> 2) * (size_t)(4 * p.W) + (size_t)((n >> 3) & 3)) * 8 + (n & 7)
                                     : (size_t)n;
            *reinterpret_cast<uint32_t*>(orow + off) = Pack2<T>::pack(fmaxf(a0, slope * a0), fmaxf(a1, slope * a1));
          }
        }
      }
  }
}

#endif  // VFI_HOST_EMU

// ---------------------------------------------------------------------------------------------
// CUDA-core checker with the SAME parameters, packed weights and epilogue: one thread per (cell, n).
// Test infrastructure for the tensor-core kernel (debug entry point only; never on the product path).
// ---------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float ld16bit(const T* p);
template <>
__device__ __forceinline__ float ld16bit<__half>(const __half* p) { return __half2float(*p); }
template <>
__device__ __forceinline__ float ld16bit<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <typename T>
__device__ __forceinline__ T cvt16bit(float v);
template <>
__device__ __forceinline__ __half cvt16bit<__half>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 cvt16bit<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <typename T>
__global__ void tapconv_ref_kernel(const __grid_constant__ TapConvParams p) {
  const size_t total = (size_t)p.B * p.H * p.W * p.n_total;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(id % p.n_total);
    size_t cell = id / p.n_total;
    const int gx = (int)(cell % p.W);
    cell /= p.W;
    const int gy = (int)(cell % p.H);
    const int b = (int)(cell / p.H);
    const int split = n / p.n_cta, nl = n - split * p.n_cta;
    const T* w = reinterpret_cast<const T*>(p.w) + (size_t)split * (p.w_bytes / 2);
    const T* in = reinterpret_cast<const T*>(p.in);
    float acc = 0.f;
    int j = 0;  // running K=16 step
    for (int e = 0; e < p.ntaps; ++e) {
      const TapEntry te = p.taps[e];
      const int y = gy + te.dy, x = gx + te.dx;
      const bool ok = y >= 0 && y < p.H && x >= 0 && x < p.W;
      for (int i = 0; i < te.nk16; ++i, ++j) {
        if (!ok) continue;
        for (int c = 0; c < 16; ++c) {
          const int cin_idx = te.chunk0 * 8 + i * 16 + c;
          const float a = ld16bit<T>(in + (((size_t)b * p.H + y) * p.W + x) * p.cin + cin_idx);
          // packed weights: [j/4][n][128-byte row], 16-byte chunks XOR-swizzled with (n & 7)
          const int chunk = (j & 3) * 2 + (c >> 3);
          const size_t widx = ((size_t)(j >> 2) * p.n_cta + nl) * 64 + (size_t)((chunk ^ (nl & 7)) * 8 + (c & 7));
          acc = fmaf(a, ld16bit<T>(w + widx), acc);
        }
      }
    }
    if (p.epi_mode == EPI_LASTCONV) {
      const int c5 = n >> 4, pos = n & 15;
      const int Hs = p.H * 4, Ws = p.W * 4;
      const size_t o = ((size_t)b * Hs + gy * 4 + (pos >> 2)) * Ws + gx * 4 + (pos & 3);
      const float v = acc + p.shift[n];
      if (c5 < 4)
        reinterpret_cast<float*>(p.out_flow)[o * 4 + c5] = v;
      else
        p.out_mask[o] = v;
    } else {
      float v = acc + p.shift[n];
      if (p.epi_mode == EPI_RESCONV) v += ld16bit<T>(in + (((size_t)b * p.H + gy) * p.W + gx) * p.cin + n);
      size_t o = out_pixel_offset(p, b, gy, gx) + n;
      if (p.out_s2d == 2) {
        const int pos = n >> 3;
        o = out_pixel_offset(p, b, gy, gx) + ((size_t)(pos >> 2) * (size_t)(4 * p.W) + (size_t)(pos & 3)) * 8 + (n & 7);
      }
      reinterpret_cast<T*>(p.out)[o] = cvt16bit<T>(p.epi_mode == EPI_BIAS ? v : lrelu02(v));
    }
  }
}

#ifndef VFI_HOST_EMU
// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
bool make_tmap(CUtensorMap* tm, CUtensorMapDataType dt, const void* base, int C, int W, int H, int B, int box_c,
               int box_w, int box_h, CUtensorMapSwizzle swz) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || !f) {
      set_error("cuTensorMapEncodeTiled is not available from this driver");
      return false;
    }
    fn = reinterpret_cast<EncodeTiledFn>(f);
  }
  // input activations as a 4-D tensor {C, W, H, B} (innermost first), 16-bit elements
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  const cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  const cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  const cuuint32_t es[4] = {1, 1, 1, 1};
  const CUresult r = fn(tm, dt, 4, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
    return false;
  }
  return true;
}

#endif  // VFI_HOST_EMU

uint32_t align_up(uint32_t v, uint32_t a) { return (v + a - 1) / a * a; }

}  // namespace

int tapconv_plan(const TapConvLayer& L, TapConvParams* pp) {
  TapConvParams& p = *pp;
  p.cin = L.cin;
  p.n_total = L.n_total;
  p.n_cta = L.n_cta;
  p.nsplit = L.nsplit;
  p.ntaps = L.ntaps;
  p.ktotal16 = L.ktotal16;
  p.halo_y0 = L.halo_y0;
  p.halo_x0 = L.halo_x0;
  p.halo_h = L.halo_h;
  p.halo_w = L.halo_w;
  p.epi_mode = L.epi_mode;
  p.out_s2d = L.out_s2d;
  for (int e = 0; e < L.ntaps; ++e) p.taps[e] = L.taps[e];
  // weights: [ceil(K16/4)][n_cta] rows of 128 B (four K=16 steps each), SWIZZLE_128B
  p.w_bytes = (uint32_t)((L.ktotal16 + 3) / 4) * (uint32_t)L.n_cta * 128u;
  // input window: one 1024-aligned region per k-block (64 channels = 128-byte rows; 32-channel tail = 64-byte rows)
  p.nkb = (L.cin + 63) / 64;
  p.ring = L.ring;
  if (L.ktotal16 > kMaxK16) return 0;
  // n_cta = the wgmma N: whole 8-row swizzle atoms of B, and a multiple of 16 with an instantiated kernel (<= 96: two
  // 64-row accumulators of n_cta fp32 columns per thread)
  if (p.nkb > kMaxKBlocks || L.n_cta > 96 || (L.n_cta & 15) || L.n_cta < 16) return 0;
  if (L.ring && ((L.cin & 63) || L.ntaps != 9 * p.nkb || L.ktotal16 != 36 * p.nkb)) return 0;
  uint32_t off = 0;
  p.tx_bytes = 0;
  if (L.ring) {
    // ring: every slot holds ONE k-block of a tile's window; p.stage_bytes / p.tx_bytes are per slot
    const uint32_t bytes = (uint32_t)L.halo_w * (uint32_t)L.halo_h * 128u;
    for (int kb = 0; kb < p.nkb; ++kb) p.kb_off[kb] = 0;
    off = align_up(bytes, 1024);
    p.tx_bytes = bytes;
  } else {
    for (int kb = 0; kb < p.nkb; ++kb) {
      const bool tail = (kb == p.nkb - 1) && (L.cin & 63);
      const uint32_t bytes = (uint32_t)L.halo_w * (uint32_t)L.halo_h * (tail ? 64u : 128u);
      p.kb_off[kb] = off;
      off += align_up(bytes, 1024);
      p.tx_bytes += bytes;
    }
  }
  p.stage_bytes = off;
  {
    // wgmma descriptor words per K=16 step (ptx.cuh): start>>4 [0,14) | LBO [16,30) ; SBO>>4 [32,46) | layout [62,64)
    // (1 = SWIZZLE_128B, 2 = SWIZZLE_64B); base_offset stays 0.
    // Ring layers list their taps k-block-major, so entries [0,36) (k-block 0) serve every k-block: the kernel adds
    // the slot address to A and kb * (9 * n_cta * 128 B) to B.
    uint4 step[kMaxK16];
    int j = 0;
    for (int e = 0; e < L.ntaps; ++e)
      for (int i = 0; i < L.taps[e].nk16; ++i, ++j) {
        const TapEntry te = L.taps[e];
        const int ch0 = te.chunk0 * 8 + 16 * i;
        const int kb = ch0 >> 6;
        const bool tail = (kb == p.nkb - 1) && (L.cin & 63);
        const uint32_t rowb = tail ? 64u : 128u;
        const uint32_t a_off = p.kb_off[kb] + (uint32_t)((te.dy - L.halo_y0) * L.halo_w + (te.dx - L.halo_x0)) * rowb +
                               (uint32_t)(ch0 - kb * 64) * 2u;
        const uint32_t b_off = (uint32_t)(j >> 2) * ((uint32_t)L.n_cta * 128u) + (uint32_t)(j & 3) * 32u;
        step[j] = make_uint4(a_off >> 4, (((uint32_t)L.halo_w * rowb) >> 4) | (tail ? kDescSw64 : kDescSw128),
                             b_off >> 4, 0u);
      }
    // group the steps into runs of run_len = 4, 2 or 1 whose descriptors advance by 32 B (2 units) per step
    const int nsteps = L.ring ? 36 : L.ktotal16;  // ring: the first k-block's entries serve every slot
    int run_len = 1;
    for (int len : {4, 2}) {
      bool ok = (nsteps % len) == 0;
      for (int r = 0; ok && r < nsteps; r += len)
        for (int i = 1; i < len; ++i)
          ok = ok && step[r + i].x == step[r].x + 2u * i && step[r + i].y == step[r].y &&
               step[r + i].z == step[r].z + 2u * i;
      if (ok) {
        run_len = len;
        break;
      }
    }
    p.run_len = run_len;
    p.nruns = nsteps / run_len;
    for (int r = 0; r < p.nruns; ++r) p.mma[r] = step[r * run_len];
  }
  p.b_hi = (1024u >> 4) | kDescSw128;  // B: SBO = 8 rows x 128 B, SWIZZLE_128B
  p.off_w = align_up(kCtrlBytes, 1024);
  p.off_a = align_up(p.off_w + p.w_bytes, 1024);
  int stages = 0;
  for (int s = kMaxStages; s >= 1; --s) {
    if (p.off_a + (uint32_t)s * p.stage_bytes <= (uint32_t)kSmemLimit) {
      stages = s;
      break;
    }
  }
  p.stages = stages;
  p.smem_bytes = p.off_a + (uint32_t)stages * p.stage_bytes;  // stage sizes are multiples of 1024
  return stages;
}

cudaError_t launch_tapconv(const TapConvLayer& L, int op_type, const void* in, void* out, float4* out_flow,
                           float* out_mask, int B, int H, int W, int num_sms, bool use_ref, cudaStream_t st) {
  TapConvParams p{};
  if (tapconv_plan(L, &p) < 1) {
    set_error("tapconv: layer does not fit in shared memory");
    return cudaErrorInvalidConfiguration;
  }
  if (L.out_s2d == 1 && ((H | W) & 1)) {
    set_error("tapconv: space-to-depth output needs even H and W");
    return cudaErrorInvalidValue;
  }
  p.in = in;
  p.out = out;
  p.out_flow = out_flow;
  p.out_mask = out_mask;
  p.w = L.w;
  p.shift = L.shift;
  p.B = B;
  p.H = H;
  p.W = W;
  p.tiles_y = (H + kTileH - 1) / kTileH;
  p.tiles_x = (W + kTileW - 1) / kTileW;
  p.ntiles = B * p.tiles_y * p.tiles_x;

#ifdef VFI_HOST_EMU
  use_ref = true;  // the host emulation has only the checker kernel
#endif
  if (use_ref) {
    const size_t total = (size_t)B * H * W * L.n_total;
    const int blocks = (int)((total + 255) / 256 < 65535 ? (total + 255) / 256 : 65535);
    if (op_type == OP_BF16)
      VFI_LAUNCH(tapconv_ref_kernel<__nv_bfloat16>, blocks, 256, 0, st, p);
    else
      VFI_LAUNCH(tapconv_ref_kernel<__half>, blocks, 256, 0, st, p);
    return cudaGetLastError();
  }
#ifdef VFI_HOST_EMU
  return cudaErrorInvalidConfiguration;
#else

  const CUtensorMapDataType dt = (op_type == OP_BF16) ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  if (L.cin >= 64 && !make_tmap(&p.tm64, dt, in, L.cin, W, H, B, 64, L.halo_w, L.halo_h, CU_TENSOR_MAP_SWIZZLE_128B))
    return cudaErrorInvalidValue;
  if (L.cin & 63) {
    if (!make_tmap(&p.tm32, dt, in, L.cin, W, H, B, 32, L.halo_w, L.halo_h, CU_TENSOR_MAP_SWIZZLE_64B))
      return cudaErrorInvalidValue;
    if (L.cin < 64) p.tm64 = p.tm32;  // a single 32-channel k-block: the 64-channel map is never used
  } else {
    p.tm32 = p.tm64;
  }
  // cps persistent CTAs per output-channel split
  int cps = num_sms / L.nsplit;
  if (cps < 1) cps = 1;
  if (cps > p.ntiles) cps = p.ntiles;
  p.ctas_per_split = cps;
  const int grid = cps * L.nsplit;
  cudaError_t err;  // (per device: set on every launch, it is a cheap driver call)
  static const bool pdl = [] {  // VFI_PDL=0: plain stream-ordered launches (A/B runs)
    const char* e = std::getenv("VFI_PDL");
    return !(e && e[0] == '0');
  }();
  auto go = [&](auto kern) -> cudaError_t {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3((unsigned)kThreads);
    cfg.dynamicSmemBytes = p.smem_bytes;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    int na = 0;
    if (pdl) {
      attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      attr[na].val.programmaticStreamSerializationAllowed = 1;
      ++na;
    }
    cfg.attrs = attr;
    cfg.numAttrs = na;
    return cudaLaunchKernelEx(&cfg, kern, p);
  };
  const bool last = (L.epi_mode == EPI_LASTCONV);
  auto pick_n = [&](auto tag, auto ring, auto lst) -> cudaError_t {
    using T = decltype(tag);
    constexpr bool R = decltype(ring)::value, LA = decltype(lst)::value;
    switch (L.n_cta) {  // tapconv_plan admits multiples of 16 up to 96
      case 16: return go(tapconv_kernel<T, R, LA, 16>);
      case 32: return go(tapconv_kernel<T, R, LA, 32>);
      case 48: return go(tapconv_kernel<T, R, LA, 48>);
      case 64: return go(tapconv_kernel<T, R, LA, 64>);
      case 80: return go(tapconv_kernel<T, R, LA, 80>);
      default: return go(tapconv_kernel<T, R, LA, 96>);
    }
  };
  auto pick = [&](auto tag) -> cudaError_t {
    using F = std::false_type;
    using Tr = std::true_type;
    if (L.ring) return last ? pick_n(tag, Tr{}, Tr{}) : pick_n(tag, Tr{}, F{});
    return last ? pick_n(tag, F{}, Tr{}) : pick_n(tag, F{}, F{});
  };
  err = (op_type == OP_BF16) ? pick(__nv_bfloat16{}) : pick(__half{});
  if (err != cudaSuccess) return err;
  return cudaGetLastError();
#endif  // VFI_HOST_EMU
}

}  // namespace vfi
