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
// Channel-major MMAs (p.cmajor, template CM: 3 x 3 convs over 64 input channels with n_cta = 64 and a staged 16-bit
// NHWC output).  The operand roles swap: the packed weights are byte for byte a K-major SWIZZLE_128B A operand (64
// output-channel rows) and the window a K-major B operand whose 8-row groups are the tile's 16 rows of 8 cells (SBO =
// halo_w * 128 B), so ONE m64n128k16 per K=16 step computes the whole tile.  Per step shared memory then supplies 2 KB
// of weights + 4 KB of window instead of 2 x (2 KB + 2 KB): with cells on M and N = 64 the two MMAs alone need all of
// an SM's shared-memory bandwidth at the tensor peak (128 B/clk against 1/16 B per MAC), channel-major three quarters
// of it.  Same products in the same K order into fp32: the outputs are bit-identical to the cell-major form (DESIGN.md
// section 5 has the measured gain).
//
// Streamed weights (p.wstream, template WS: the wide ResConvs, c = 96 / 128 / 192, block 1's lastconv, c = 128, and
// the 4.26 feature conv at c = 128 / 192).  A resident weight slice of such a layer leaves room for only 16 - 64
// output channels per CTA, so every tile's window would be read from L2 and shared memory once per output-channel
// split, and the narrow wgmma N leaves the tensor cores waiting on shared memory (an SS wgmma reads its 2 KB A block
// whatever its N).  Here the window of a tile is staged once with all its k-blocks and held until the epilogue, and the
// weights stream through a ring of slots of four K=16 steps each (the packed [K16 / 4][n_cta][128 B] rows, one bulk
// copy per slot) fed by a second producer warp: n_cta = 96 / 128 / 96 output channels per CTA for the ResConvs, all
// 80 / 128 columns for lastconv / the feature conv.  Both MMA warpgroups take a tile each and consume every slot in
// step, so one weight fill from L2 feeds 256 cells.  The K=16 steps keep the order of the layer's tap list (k-block-major at c = 128 / 192,
// tap-major at c = 96, whose two extra zero-weight steps only complete the last slot): every output is the same fp32
// sum in the same order as with resident weights.
//
// Warp roles (288 threads, 1 CTA/SM, persistent over tiles; WS: 320):
//   warpgroups 0, 1 : MMA + epilogue.  Warpgroup w takes the CTA's tiles w, w + 2, ... and keeps the whole tile's
//                     accumulators (2 x 64 rows x n_cta columns, fp32) in registers, so one warpgroup's epilogue
//                     overlaps the other's MMAs: +shift (held in registers for the launch), +residual (ResConv:
//                     ldmatrix from the tile's still-held window stage, then the stage is released), LeakyReLU,
//                     16-bit; NHWC outputs are stmatrix'ed into a swizzled per-warpgroup staging tile and leave as TMA
//                     tensor stores (one thread, clipped at the image border); lastconv writes whole float4 flow
//                     texels, the space-to-depth forms direct stores.
//   warp 8          : one elected lane: weight bulk copy, then one 4-D TMA tensor copy per k-block and tile
//   warp 9 (WS)     : one elected lane: one bulk copy per weight slot, the whole weight stream once per pair of tiles
#include <algorithm>
#include <type_traits>

#include "ptx.cuh"
#include "vfi_internal.h"

namespace vfi {

namespace {

constexpr int kMaxStages = 6;   // window stages
constexpr int kMaxWSlots = 8;   // streamed weight slots
struct Ctrl {
  uint64_t w_full;
  uint64_t a_full[kMaxStages][2];  // [stage][consuming warpgroup]
  uint64_t a_empty[kMaxStages];
  uint64_t ws_full[kMaxWSlots];    // WS: weight slot filled (bulk-copy bytes)
  uint64_t ws_empty[kMaxWSlots];   // WS: every warp of both MMA warpgroups has read the slot
};
constexpr uint32_t kCtrlBytes = 512;
constexpr int kMmaGroups = 2, kTmaWarp = 8, kWeightWarp = 9, kThreads = 128 * kMmaGroups + 32;
constexpr int kThreadsWS = kThreads + 32;
static_assert(sizeof(Ctrl) <= kCtrlBytes, "control block");
constexpr int kCmRuns = 9, kCmRunLen = 4;  // channel-major MMA issue: 9 taps x 4 K=16 steps (64 input channels)

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

// Channels per TMA store box of a 16-bit NHWC output: the widest of 64 / 32 / 16 that divides the CTA's n_cta, so the
// box row is 128 / 64 / 32 bytes and uses the swizzle of that width (conflict-free stmatrix into the staging tile).
__host__ __device__ constexpr int store_box_c(int n_cta) { return n_cta % 64 == 0 ? 64 : n_cta % 32 == 0 ? 32 : 16; }

uint32_t align_up(uint32_t v, uint32_t a) { return (v + a - 1) / a * a; }

#ifndef VFI_HOST_EMU  // (tests/host_emu runs the RIFE schedule on the CPU with the checker kernel; no wgmma there)
// Byte offset of 16-byte chunk `chunk` of row `row` in a 1024-aligned region of rowb-byte rows (32, 64 or 128) laid out
// by TMA with the swizzle of that width: address bits [4, 4 + log2(rowb / 16)) are XORed with bits [7, ...).
__device__ __forceinline__ uint32_t swz_off(uint32_t row, uint32_t chunk, uint32_t rowb) {
  const uint32_t o = row * rowb + chunk * 16u;
  return o ^ (((o >> 7) & (rowb / 16u - 1u)) << 4);
}

// Walks the tiles of one CTA (t = first, first + cps, ...) keeping (image, tile row, tile column) incrementally
// instead of two integer divisions per tile and role.
struct TileIter {
  int b, ty, tx, db, dy, dx, tiles_x, tiles_y;
  template <class P>
  __device__ __forceinline__ TileIter(const P& p, int first, int step) {
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
// LBO = 1) of the window and of the weights of this k-block.  CM: one m64n128 per step, weights as A and the window as
// B; its accumulator d[4 j + 2 h + c] (tile row j = 0..15) is acc[j / 8][4 (j % 8) + 2 h + c].  The channel-major
// layers are 3 x 3 convs over 64 channels (tapconv_plan: kCmRuns runs of kCmRunLen steps), so their 36 MMAs are issued
// as straight-line code: with no loop back-edge between them ptxas keeps them one chain behind a single
// warpgroup.arrive instead of injecting an arrive in front of every MMA and ending each one's scoreboard group.
template <int N, bool CM, typename T>
__device__ __forceinline__ void issue_window(const TapConvParams& p, float (&acc)[2][N / 2], uint32_t a_base,
                                             uint32_t b_base) {
  if constexpr (CM) {
#pragma unroll
    for (int r = 0; r < kCmRuns; ++r) {
      const uint4 d = p.mma[r];
      const uint64_t w64 = ((uint64_t)p.b_hi << 32) | (uint64_t)(b_base + d.z);
      const uint64_t x64 = ((uint64_t)d.y << 32) | (uint64_t)(a_base + d.x);
#pragma unroll
      for (int i = 0; i < kCmRunLen; ++i)
        wgmma_ss<128, T>(&acc[0][0], w64 + 2u * i, x64 + 2u * i, (r | i) ? 1u : 0u);
    }
    return;
  }
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
        wgmma_ss<N, T>(acc[h], a64, b64, (r | i) ? 1u : 0u);
        a64 += 2;
        b64 += 2;
      }
    }
  }
}

// WS: the MMAs of weight slot `grp` (K=16 steps 4 grp .. 4 grp + 3; tapconv_plan admits K16 % 4 == 0 only) for both
// 64-row halves of the tile.  p.mma[j] is step j's window descriptor; its weights start 32 B * (j % 4) into the slot.
// Straight-line: a conditional exit between the MMAs makes ptxas serialize every wgmma of the kernel (C7520).
template <int N, typename T>
__device__ __forceinline__ void issue_wslot(const TapConvParams& p, float (&acc)[2][N / 2], uint32_t a_base,
                                            uint32_t b_base, int grp) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int j = 4 * grp + i;
    const uint4 d = p.mma[j];
    const uint32_t half_off = 8u * (d.y & 0x3fffu);
    const uint64_t b64 = ((uint64_t)p.b_hi << 32) | (uint64_t)(b_base + 2u * i);
#pragma unroll
    for (int h = 0; h < 2; ++h)
      wgmma_ss<N, T>(acc[h], ((uint64_t)d.y << 32) | (uint64_t)(a_base + d.x + (uint32_t)h * half_off), b64,
                     j ? 1u : 0u);
  }
}

// Staged 16-bit output of one 64-row accumulator half: this warp's tile rows `row` and `row + 1` (d[4 j + 2 e + c] = tile
// row row + e, column lane / 4, channel 8 j + c2 + c), through max(a, slope * a) and rounded to 16 bits, stmatrix'ed into
// a staging tile of N / store_box_c(N) boxes of box_bytes each, swizzled like the box rows.
template <int N, typename T>
__device__ __forceinline__ void stage_rows(const float (&a)[N / 2], uint32_t out_smem, uint32_t box_bytes, int row, int lane,
                                           float slope) {
  constexpr int kBoxC = store_box_c(N);
  constexpr uint32_t kBoxRow = 2u * kBoxC;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const uint32_t pix = (uint32_t)((row + e) * kTileW + (lane & 7));
#pragma unroll
    for (int jb = 0; jb < N / 8; jb += 4) {
      const bool x4 = N / 8 - jb >= 4;
      const int col = 8 * (jb + (x4 ? (lane >> 3) : ((lane >> 3) & 1)));
      const uint32_t addr = out_smem + (uint32_t)(col / kBoxC) * box_bytes + swz_off(pix, (uint32_t)(col % kBoxC) >> 3, kBoxRow);
      uint32_t r[4];
#pragma unroll
      for (int i = 0; i < (x4 ? 4 : 2); ++i) {
        const float a0 = a[4 * (jb + i) + 2 * e], a1 = a[4 * (jb + i) + 2 * e + 1];
        r[i] = Pack2<T>::pack(fmaxf(a0, slope * a0), fmaxf(a1, slope * a1));
      }
      if (x4)
        stsm_x4(addr, r);
      else
        stsm_x2(addr, r);
    }
  }
}

template <typename T, bool LAST, int N, bool CM, bool WS>
__global__ void __launch_bounds__(WS ? kThreadsWS : kThreads, 1) tapconv_kernel(const __grid_constant__ TapConvParams p) {
  static_assert(!CM || (N == 64 && !LAST), "channel-major: 64 output channels, 16-bit output");
  static_assert(!WS || !CM, "streamed weights: cells on M");
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
  const uint32_t bar_wsfull = smem_base + offsetof(Ctrl, ws_full);
  const uint32_t bar_wsempty = smem_base + offsetof(Ctrl, ws_empty);
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
    if (WS)
      for (int s = 0; s < p.w_slots; ++s) {
        mbar_init(bar_wsfull + 8 * s, 1);
        mbar_init(bar_wsempty + 8 * s, 4 * kMmaGroups);
      }
    mbar_fence_init();
  }
  __syncthreads();

  if (WS && warp == kWeightWarp) {
    // ======================================================= weight producer: the slots of every pass of two tiles
    if (lane == 0) {
      const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(p.w) + (size_t)split * p.w_bytes;
      uint32_t slot = 0, ph = 0;
      for (int q = 0; q < (my_tiles + 1) / 2; ++q)
        for (int grp = 0; grp < p.w_groups; ++grp) {
          mbar_wait(bar_wsempty + 8 * slot, ph ^ 1u);
          mbar_arrive_expect_tx(bar_wsfull + 8 * slot, p.w_slot_bytes);
          bulk_g2s(w_smem + slot * p.w_slot_bytes, wsrc + (size_t)grp * p.w_slot_bytes, p.w_slot_bytes,
                   bar_wsfull + 8 * slot);
          if (++slot == (uint32_t)p.w_slots) {
            slot = 0;
            ph ^= 1u;
          }
        }
    }
    return;
  }
  if (warp == kTmaWarp) {
    // ======================================================= TMA producer (one thread feeds the whole pipeline)
    if (lane == 0) {
      if (!WS) {
        mbar_arrive_expect_tx(bar_w, p.w_bytes);
        const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(p.w) + (size_t)split * p.w_bytes;
        for (uint32_t off = 0; off < p.w_bytes; off += 32768u)
          bulk_g2s(w_smem + off, wsrc + off, min(32768u, p.w_bytes - off), bar_w);
      }
      // weights do not depend on the previous kernel; its output (our input tensor) does
      asm volatile("griddepcontrol.wait;" ::: "memory");
      TileIter it(p, first, tstep);
      uint32_t stage = 0, eph = 1;  // window stage and the parity of its "empty" barrier
      for (int k = 0; k < my_tiles; ++k, it.next()) {
        const int gy0 = it.ty * kTileH + p.halo_y0, gx0 = it.tx * kTileW + p.halo_x0;
        const uint32_t full = bar_afull + 16 * stage + 8 * (k & 1);  // tile k goes to warpgroup k % 2
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
    return;
  }

  // ========================================================= MMA + epilogue warpgroups
  // Warpgroup g consumes the stages of tiles g, g + 2, ... through its own "full" barrier of each stage: the fills a
  // warpgroup waits for on one barrier are its own, in order, so a parity wait never confuses an older phase with the
  // one it wants (a stage shared by both warpgroups would, with one or an odd number of stages).
  const int g = warp >> 2;
  const int wq = warp & 3;  // warp of the warpgroup: rows 16 wq .. 16 wq + 15 of each 64-row half
  const int px = lane >> 2;             // tile column of this thread's accumulator rows
  const int c2 = 2 * (lane & 3);        // first of this thread's two columns in every 8-column block
  // the CTA's output-channel slice is fixed: its shift values stay in registers for the whole launch (channel-major:
  // this thread's two channels 16 wq + lane / 4, +8; WS: read per tile, the registers hold the N = 128 accumulators)
  float2 sh[(CM || WS) ? 1 : N / 8];
  if constexpr (CM) {
    const int ch = n0 + 16 * wq + (lane >> 2);
    sh[0] = make_float2(__ldg(p.shift + ch), __ldg(p.shift + ch + 8));
  } else if constexpr (!WS) {
#pragma unroll
    for (int j = 0; j < N / 8; ++j) sh[j] = __ldg(reinterpret_cast<const float2*>(p.shift + n0 + 8 * j + c2));
  }
  // the previous kernel may still be reading the buffer we store to (ping-pong): every storing thread orders itself
  // after the previous grid
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (!WS) mbar_wait(bar_w, 0);
  const uint32_t a_lo0 = (1u << 16) | (a_smem >> 4);  // LBO(=1) | start address, 16-byte units
  const uint32_t b_lo0 = (1u << 16) | (w_smem >> 4);
  const uint32_t stage_units = p.stage_bytes >> 4;
  uint32_t stage = 0, ph_bits = 0;  // window stage; bit s: parity of this warpgroup's next wait on stage s
  auto advance = [&](uint32_t n) {
    stage += n;
    while (stage >= (uint32_t)S) stage -= (uint32_t)S;
  };
  auto wait_full = [&]() {
    mbar_wait(bar_afull + 16 * stage + 8 * (uint32_t)g, (ph_bits >> stage) & 1u);
    ph_bits ^= 1u << stage;
  };
  advance((uint32_t)g);
  const float slope = (p.epi_mode == EPI_BIAS) ? 1.f : 0.2f;  // max(a, slope * a): LeakyReLU(0.2), or no activation
  // TMA-stored outputs: each warpgroup packs its tile into its own staging tile, [box][16 x 8 pixels][kBoxC channels]
  // swizzled like the box rows, and one thread stores it as N / kBoxC tensor boxes
  constexpr int kBoxC = store_box_c(N);
  constexpr uint32_t kBoxRow = 2u * kBoxC, kBoxBytes = (uint32_t)(kTileH * kTileW) * kBoxRow;
  const bool tma_out = CM || (!LAST && p.out_stage_bytes != 0);  // (channel-major layers always stage their output)
  const bool leader = (threadIdx.x & 127) == 0;  // issues and waits for the warpgroup's bulk groups
  const uint32_t out_smem = smem_base + p.off_out + (uint32_t)g * p.out_stage_bytes;
  float acc[2][N / 2];
  uint32_t wslot = 0, wph = 0;  // WS: next weight slot and the parity of its "full" barrier
  const uint32_t w_slot_units = p.w_slot_bytes >> 4;
  auto next_wslot = [&]() {
    if (++wslot == (uint32_t)p.w_slots) {
      wslot = 0;
      wph ^= 1u;
    }
  };

  TileIter it(p, first + g * tstep, kMmaGroups * tstep);
  for (int k = g; k < my_tiles; k += kMmaGroups, it.next()) {
    if (WS) {
      wait_full();
      const uint32_t a_base = a_lo0 + stage * stage_units;
      uint32_t prev = 0;
      for (int grp = 0; grp < p.w_groups; ++grp) {
        mbar_wait(bar_wsfull + 8 * wslot, wph);
        wgmma_fence();
        issue_wslot<N, T>(p, acc, a_base, b_lo0 + wslot * w_slot_units, grp);
        wgmma_commit();
        if (grp > 0) {  // the previous slot's MMAs have read it
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_wsempty + 8 * prev);
        }
        prev = wslot;
        next_wslot();
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_wsempty + 8 * prev);
      if (!residual && lane == 0) mbar_arrive(bar_aempty + 8 * stage);
    } else {
      wait_full();
      wgmma_fence();
      issue_window<N, CM, T>(p, acc, a_lo0 + stage * stage_units, b_lo0);
      wgmma_commit();
      wgmma_wait<0>();
      if (!residual) {  // window free once the MMAs have read it (ResConv reads its residual from it first)
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_aempty + 8 * stage);
      }
    }
    acc_fence(acc[0]);
    acc_fence(acc[1]);

    // ---- epilogue from the accumulator registers: d[h][4 j + 2 e + c] = tile row 8 h + 2 wq + e, column 8 j + c2 + c
    // channel-major: acc[jh][4 jl + 2 h + c] = channel 16 wq + lane / 4 + 8 h of tile row 8 jh + jl, column c2 + c
    const int b = it.b;
    const int gy0 = it.ty * kTileH, gx0 = it.tx * kTileW;
    if constexpr (CM) {
#pragma unroll
      for (int jh = 0; jh < 2; ++jh)
#pragma unroll
        for (int jl = 0; jl < 8; ++jl) {
          acc[jh][4 * jl] += sh[0].x;
          acc[jh][4 * jl + 1] += sh[0].x;
          acc[jh][4 * jl + 2] += sh[0].y;
          acc[jh][4 * jl + 3] += sh[0].y;
        }
    } else {
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
          float2 s;
          if constexpr (WS)
            s = __ldg(reinterpret_cast<const float2*>(p.shift + n0 + 8 * j + c2));
          else
            s = sh[j];
          acc[h][4 * j] += s.x;
          acc[h][4 * j + 1] += s.y;
          acc[h][4 * j + 2] += s.x;
          acc[h][4 * j + 3] += s.y;
        }
    }
    if (residual) {
      // the residual is the centre of the tile's staged window, still held: channel n of window pixel
      // (y - halo_y0, x - halo_x0), read as 8 x 8 (pixel, channel) matrices straight into the accumulator layout
      const uint32_t win = a_smem + stage * p.stage_bytes;
      if constexpr (CM) {
        // transposed reads: matrix i = lane / 8 is tile row 8 jh + 2 jp + i / 2 (8 cells) x channels 16 wq + 8 (i % 2)
        const int i = lane >> 3;
        const int ch = n0 + 16 * wq + 8 * (i & 1);
        const int kb = ch >> 6;
        const uint32_t rowb = (has_tail && kb == p.nkb - 1) ? 64u : 128u;
#pragma unroll
        for (int jh = 0; jh < 2; ++jh)
#pragma unroll
          for (int jp = 0; jp < 4; ++jp) {
            const int row = 8 * jh + 2 * jp + (i >> 1);
            const uint32_t pix = (uint32_t)((row - p.halo_y0) * p.halo_w + (lane & 7) - p.halo_x0);
            uint32_t r[4];
            ldsm_x4_t(win + p.kb_off[kb] + swz_off(pix, (uint32_t)(ch & 63) >> 3, rowb), r);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float2 rf = Pack2<T>::unpack(r[q]);
              acc[jh][4 * (2 * jp + (q >> 1)) + 2 * (q & 1)] += rf.x;
              acc[jh][4 * (2 * jp + (q >> 1)) + 2 * (q & 1) + 1] += rf.y;
            }
          }
      } else {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const uint32_t pix = (uint32_t)((8 * h + 2 * wq + e - p.halo_y0) * p.halo_w + (lane & 7) - p.halo_x0);
#pragma unroll
            for (int jb = 0; jb < N / 8; jb += 4) {
              const bool x4 = N / 8 - jb >= 4;  // N / 8 is even: an x2 tail at most
              const int ch = n0 + 8 * (jb + (x4 ? (lane >> 3) : ((lane >> 3) & 1)));
              const int kb = ch >> 6;
              const uint32_t rowb = (has_tail && kb == p.nkb - 1) ? 64u : 128u;
              const uint32_t addr = win + p.kb_off[kb] + swz_off(pix, (uint32_t)(ch & 63) >> 3, rowb);
              uint32_t r[4];
              if (x4)
                ldsm_x4(addr, r);
              else
                ldsm_x2(addr, r);
#pragma unroll
              for (int i = 0; i < (x4 ? 4 : 2); ++i) {
                const float2 rf = Pack2<T>::unpack(r[i]);
                acc[h][4 * (jb + i) + 2 * e] += rf.x;
                acc[h][4 * (jb + i) + 2 * e + 1] += rf.y;
              }
            }
          }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_aempty + 8 * stage);
    }
    advance((uint32_t)kMmaGroups);

    if (tma_out) {
      if (leader) bulk_wait_read<0>();  // the previous tile's stores have read the staging tile
      named_bar_sync(1 + g, 128);
      if constexpr (CM) {
        // transposed stores: matrix i = lane / 8 is tile row 8 jh + 2 jp + i / 2 x channels 16 wq + 8 (i % 2) (one box)
        const int i = lane >> 3;
        const uint32_t chunk = (uint32_t)(2 * wq + (i & 1));
#pragma unroll
        for (int jh = 0; jh < 2; ++jh)
#pragma unroll
          for (int jp = 0; jp < 4; ++jp) {
            const uint32_t pix = (uint32_t)((8 * jh + 2 * jp + (i >> 1)) * kTileW + (lane & 7));
            uint32_t r[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float a0 = acc[jh][4 * (2 * jp + (q >> 1)) + 2 * (q & 1)];
              const float a1 = acc[jh][4 * (2 * jp + (q >> 1)) + 2 * (q & 1) + 1];
              r[q] = Pack2<T>::pack(fmaxf(a0, slope * a0), fmaxf(a1, slope * a1));
            }
            stsm_x4_t(out_smem + swz_off(pix, chunk, kBoxRow), r);
          }
      } else {
#pragma unroll
        for (int h = 0; h < 2; ++h) stage_rows<N, T>(acc[h], out_smem, kBoxBytes, 8 * h + 2 * wq, lane, slope);
      }
      fence_proxy_async();  // the generic-proxy staging writes before the TMA engine reads them
      named_bar_sync(1 + g, 128);
      if (leader) {
#pragma unroll
        for (int s = 0; s < N / kBoxC; ++s)
          tma_store_4d(&p.tm_out, out_smem + (uint32_t)s * kBoxBytes, n0 + s * kBoxC, gx0, gy0, b);
        bulk_commit();
      }
      continue;
    }

    // ---- direct stores: lastconv's fp32 planes and the space-to-depth / sub-pixel patch forms
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int gy = gy0 + 8 * h + 2 * wq + e, gx = gx0 + px;
        if (gy >= p.H || gx >= p.W) continue;
        if (LAST) {
          // column n = c5*16 + pos: component c5 (4 flow + mask) of sub-pixel pos = y4*4 + x4 of this cell's 4x4 patch
          const int Hs = p.H * 4, Ws = p.W * 4;
          if (N == 80) {
            // all 80 columns in this CTA (n0 = 0): columns j = 2 c5 + s of this thread hold component c5 of sub-pixels
            // (y4, x4) = (2 s + c2 / 4, c2 % 4 + c), so it writes whole float4 flow texels and float2 mask pairs
#pragma unroll
            for (int s = 0; s < 2; ++s) {
              const size_t o = ((size_t)b * Hs + (gy * 4 + 2 * s + (c2 >> 2))) * Ws + gx * 4 + (c2 & 3);
#pragma unroll
              for (int c = 0; c < 2; ++c)
                p.out_flow[o + c] = make_float4(acc[h][4 * s + 2 * e + c], acc[h][4 * (2 + s) + 2 * e + c],
                                                acc[h][4 * (4 + s) + 2 * e + c], acc[h][4 * (6 + s) + 2 * e + c]);
              *reinterpret_cast<float2*>(p.out_mask + o) =
                  make_float2(acc[h][4 * (8 + s) + 2 * e], acc[h][4 * (8 + s) + 2 * e + 1]);
            }
            continue;
          }
#pragma unroll
          for (int j = 0; j < N / 8; ++j) {
            const int n = n0 + 8 * j + c2;
            const int c5 = n >> 4, pos = n & 15;  // n even: n + 1 is the next sub-pixel of the same patch row
            const size_t o = ((size_t)b * Hs + (gy * 4 + (pos >> 2))) * Ws + gx * 4 + (pos & 3);
            const float v0 = acc[h][4 * j + 2 * e], v1 = acc[h][4 * j + 2 * e + 1];
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
#pragma unroll
          for (int j = 0; j < N / 8; ++j) {
            const int n = n0 + 8 * j + c2;
            const float a0 = acc[h][4 * j + 2 * e], a1 = acc[h][4 * j + 2 * e + 1];
            // patch form: columns n = sub-pixel (n >> 3) x channel (n & 7)
            const size_t off = patch ? ((size_t)((n >> 3) >> 2) * (size_t)(4 * p.W) + (size_t)((n >> 3) & 3)) * 8 + (n & 7)
                                     : (size_t)n;
            *reinterpret_cast<uint32_t*>(orow + off) = Pack2<T>::pack(fmaxf(a0, slope * a0), fmaxf(a1, slope * a1));
          }
        }
      }
  }
  if (WS && (my_tiles & 1) && g == 1) {  // the last pass has no tile for warpgroup 1: it still releases every slot
    for (int grp = 0; grp < p.w_groups; ++grp) {
      mbar_wait(bar_wsfull + 8 * wslot, wph);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_wsempty + 8 * wslot);
      next_wslot();
    }
  }
  if (tma_out && leader) bulk_wait<0>();  // the CTA's last stores have landed before it exits
}

#endif  // VFI_HOST_EMU

// ---------------------------------------------------------------------------------------------
// conv0.0 -> conv0.1 of a full-resolution arch-4.6 block as one launch (conv0_fused_kernel): conv0.0's output never
// leaves the SM.  One tile = 8 x 8 conv0.1 outputs (quarter-resolution cells).  conv0.1 reads the 9 x 9 conv0.0 cells
// [y0 - 1, y0 + 7] x [x0 - 1, x0 + 7] (its stride-2 taps are dy, dx in {-1, 0}), i.e. 18 x 18 conv0.0 outputs in
// space-to-depth form, which read the 19 x 19 block-input cells from (2 y0 - 3, 2 x0 - 3): one TMA box, zero-filled
// outside the image as for the unfused conv0.0.
//   conv0.0 runs cell-major on that window taken as ONE row of kC0XW-cell rows: output (wr, wc) of the window
//   (1 <= wr, wc <= 18) is window row L = wr * kC0XW + wc, and its tap (dy, dx) window row L + dy * kC0XW + dx, so each
//   m64n32 MMA covers 64 consecutive L (SBO = 8 rows x 128 B) and kC0MB of them cover L in [kC0XW + 1, 18 kC0XW + 18]
//   (the wc = 0 column and the rows read past the loaded box give outputs that are dropped).  Its epilogue (shift,
//   LeakyReLU, 16-bit) writes the conv0.1 window exactly as TMA would have staged conv0.0's space-to-depth output: two
//   SWIZZLE_128B k-blocks (sub-rows 0 and 1) of 9 x 9 cells x 128 B, and zeros for cells outside the grid (conv0.1's
//   padding).  conv0.1 then runs its planned tap descriptors on that window (one m64 row block) and leaves through the
//   staged TMA store.  Same products in the same K order into fp32 and the same roundings as the two launches.
// Shared memory: control block, both layers' weights (resident for the launch), and per MMA warpgroup its x window, its
// conv0.1 window and its output staging tile.  Warpgroup g takes the CTA's tiles g, g + 2, ...; the producer refills a
// warpgroup's x window as soon as that warpgroup's conv0.0 MMAs have read it, so one fill is in flight while both compute.
constexpr int kC0XW = 19;                                // x window: 19 x 19 cells of 64 channels (128 B)
constexpr int kC0MB = 6;                                 // conv0.0 m64 row blocks: L in [20, 20 + 384)
constexpr uint32_t kC0XBox = kC0XW * kC0XW * 128u;       // TMA bytes of one x window
constexpr uint32_t kC0XBytes = (kC0XW + 1 + 64 * kC0MB) * 128u;  // rows the conv0.0 MMAs address (past the box: unused)
constexpr int kC0Tile = 8;                               // conv0.1 tile: 8 x 8 cells
constexpr uint32_t kC0OutBytes = kC0Tile * kC0Tile * 128u;  // 64 channels x 16 bit per cell

struct alignas(64) Conv0Params {
  CUtensorMap tm_x;    // block input {64, W2, H2, B}, box {64, 19, 19, 1}, SWIZZLE_128B
  CUtensorMap tm_out;  // conv0.1 output {64, W4, H4, B}, box {64, 8, 8, 1}, SWIZZLE_128B
  const void* w0;      // conv0.0 / conv0.1 packed weights and shifts (their TapConvLayers)
  const void* w1;
  const float* shift0;
  const float* shift1;
  int B, H4, W4;  // conv0.1 grid (conv0.0's: 2 H4 x 2 W4)
  int tiles_x, tiles_y, ntiles, ctas;
  uint32_t w0_bytes, w1_bytes;
  uint32_t off_w0, off_w1, off_wg, wg_bytes, off_c00, c00_kb1, off_out, smem_bytes;
  uint32_t b_hi;  // weight (B) descriptor high word of both layers
  uint4 mma0[9];  // conv0.0 steps {A offset from the x window, A high word, B offset, 0}, 16-byte units
  uint4 mma1[9];  // conv0.1 runs of two steps {A offset from the conv0.1 window, A high word, B offset, 0}
};

// Both layers' shapes as the kernel hard-codes them: conv0.0 64 -> 32 channels as 9 one-step taps, conv0.1 128 -> 64 as
// 9 two-step runs, each in one output-channel split.  Fills the shared-memory layout and descriptors; false otherwise.
bool conv0_fused_layout(const TapConvLayer& L0, const TapConvLayer& L1, Conv0Params* pp) {
  Conv0Params& p = *pp;
  if (L0.cin != 64 || L0.n_total != 32 || L0.nsplit != 1 || L0.ntaps != 9 || L0.ktotal16 != 9 || L0.out_s2d != 1 ||
      L0.epi_mode != EPI_BIAS_LRELU || L1.cin != 128 || L1.n_total != 64 || L1.nsplit != 1 || L1.out_s2d != 0 ||
      L1.epi_mode != EPI_BIAS_LRELU || L1.halo_y0 != -1 || L1.halo_x0 != -1 || L1.halo_w != kC0Tile + 1)
    return false;
  for (int e = 0; e < 9; ++e)
    if (L0.taps[e].nk16 != 1 || L0.taps[e].dy < -1 || L0.taps[e].dy > 0 || L0.taps[e].dx < -1 || L0.taps[e].dx > 0)
      return false;
  // conv0.1's window: its layer planned over a 9-row window (the descriptors depend on the rows only through kb_off)
  TapConvLayer L1w = L1;
  L1w.halo_h = kC0Tile + 1;
  TapConvParams q{};
  if (tapconv_plan(L1w, &q) < 1 || q.nkb != 2 || q.nruns != 9 || q.run_len != 2) return false;
  p.w0_bytes = 3u * 32u * 128u;  // ceil(9 / 4) rows of four K=16 steps x 32 columns
  p.w1_bytes = q.w_bytes;
  p.b_hi = q.b_hi;
  for (int r = 0; r < 9; ++r) p.mma1[r] = q.mma[r];
  p.c00_kb1 = q.kb_off[1];
  for (int j = 0; j < 9; ++j) {
    const TapEntry te = L0.taps[j];
    const uint32_t a_off = (uint32_t)(kC0XW + 1 + te.dy * kC0XW + te.dx) * 128u + (uint32_t)te.chunk0 * 16u;
    const uint32_t b_off = (uint32_t)(j >> 2) * (32u * 128u) + (uint32_t)(j & 3) * 32u;
    p.mma0[j] = make_uint4(a_off >> 4, (1024u >> 4) | kDescSw128, b_off >> 4, 0u);
  }
  p.off_w0 = align_up(kCtrlBytes, 1024);
  p.off_w1 = align_up(p.off_w0 + p.w0_bytes, 1024);
  p.off_wg = align_up(p.off_w1 + p.w1_bytes, 1024);
  p.off_c00 = align_up(kC0XBytes, 1024);
  p.off_out = p.off_c00 + q.stage_bytes;
  p.wg_bytes = p.off_out + kC0OutBytes;
  p.smem_bytes = p.off_wg + (uint32_t)kMmaGroups * p.wg_bytes;
  return p.smem_bytes <= (uint32_t)kSmemLimit;
}

#ifndef VFI_HOST_EMU
template <typename T>
__global__ void __launch_bounds__(kThreads, 1) conv0_fused_kernel(const __grid_constant__ Conv0Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  asm volatile("griddepcontrol.launch_dependents;");  // (programmatic dependent launch, as tapconv_kernel)
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int first = (int)blockIdx.x;
  const int tstep = p.ctas;
  const int my_tiles = (p.ntiles - first + tstep - 1) / tstep;
  const uint32_t smem_base = smem_u32(smem);
  // control block: weights full, then per warpgroup its x window's "full" and "empty" barriers
  const uint32_t bar_w = smem_base, bar_full = smem_base + 8, bar_empty = smem_base + 8 + 8 * kMmaGroups;
  const uint32_t w0_smem = smem_base + p.off_w0, w1_smem = smem_base + p.off_w1;
  if (threadIdx.x == 0) {
    mbar_init(bar_w, 1);
    for (int g = 0; g < kMmaGroups; ++g) {
      mbar_init(bar_full + 8 * g, 1);
      mbar_init(bar_empty + 8 * g, 4);  // the four warps of the warpgroup
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == kTmaWarp) {
    if (lane == 0) {
      mbar_arrive_expect_tx(bar_w, p.w0_bytes + p.w1_bytes);
      bulk_g2s(w0_smem, p.w0, p.w0_bytes, bar_w);
      for (uint32_t off = 0; off < p.w1_bytes; off += 32768u)
        bulk_g2s(w1_smem + off, reinterpret_cast<const uint8_t*>(p.w1) + off, min(32768u, p.w1_bytes - off), bar_w);
      asm volatile("griddepcontrol.wait;" ::: "memory");
      TileIter it(p, first, tstep);
      // bit g: parity of the next "empty" wait on warpgroup g's window (1: the first fill of each window needs no wait)
      uint32_t eph = (1u << kMmaGroups) - 1u;
      for (int k = 0; k < my_tiles; ++k, it.next()) {
        const int g = k & 1;
        mbar_wait(bar_empty + 8 * g, (eph >> g) & 1u);
        eph ^= 1u << g;
        mbar_arrive_expect_tx(bar_full + 8 * g, kC0XBox);
        tma_load_4d(smem_base + p.off_wg + (uint32_t)g * p.wg_bytes, &p.tm_x, bar_full + 8 * g, 0,
                    2 * kC0Tile * it.tx - 3, 2 * kC0Tile * it.ty - 3, it.b);
      }
    }
    return;
  }

  const int g = warp >> 2;
  const int wq = warp & 3;
  const int px = lane >> 2;
  const int c2 = 2 * (lane & 3);
  float2 sh0[4], sh1[8];
#pragma unroll
  for (int j = 0; j < 4; ++j) sh0[j] = __ldg(reinterpret_cast<const float2*>(p.shift0 + 8 * j + c2));
#pragma unroll
  for (int j = 0; j < 8; ++j) sh1[j] = __ldg(reinterpret_cast<const float2*>(p.shift1 + 8 * j + c2));
  asm volatile("griddepcontrol.wait;" ::: "memory");
  mbar_wait(bar_w, 0);
  const uint32_t region = smem_base + p.off_wg + (uint32_t)g * p.wg_bytes;
  const uint32_t c00 = region + p.off_c00, out_smem = region + p.off_out;
  const uint32_t x_lo = (1u << 16) | (region >> 4), c00_lo = (1u << 16) | (c00 >> 4);
  const uint32_t b0_lo = (1u << 16) | (w0_smem >> 4), b1_lo = (1u << 16) | (w1_smem >> 4);
  const bool leader = (threadIdx.x & 127) == 0;
  const int H2 = 2 * p.H4, W2 = 2 * p.W4;
  uint32_t fph = 0;
  float acc0[kC0MB][16];
  float acc1[32];

  TileIter it(p, first + g * tstep, kMmaGroups * tstep);
  for (int k = g; k < my_tiles; k += kMmaGroups, it.next()) {
    mbar_wait(bar_full + 8 * g, fph);
    fph ^= 1u;
    // ---- conv0.0: 9 K=16 steps (the layer's tap order), each over the kC0MB row blocks
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 9; ++j) {
      const uint4 d = p.mma0[j];
      const uint64_t b64 = ((uint64_t)p.b_hi << 32) | (uint64_t)(b0_lo + d.z);
#pragma unroll
      for (int mb = 0; mb < kC0MB; ++mb)
        wgmma_ss<32, T>(acc0[mb], ((uint64_t)d.y << 32) | (uint64_t)(x_lo + d.x + 512u * mb), b64, j ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty + 8 * g);  // the x window may refill
#pragma unroll
    for (int mb = 0; mb < kC0MB; ++mb) acc_fence(acc0[mb]);

    // ---- conv0.0 epilogue into the conv0.1 window: row m = 16 wq + 8 e + px of block mb is window row L
    const int hy0 = 2 * kC0Tile * it.ty - 3, hx0 = 2 * kC0Tile * it.tx - 3;  // x / conv0.0 cell of window (0, 0)
#pragma unroll
    for (int mb = 0; mb < kC0MB; ++mb)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int L = kC0XW + 1 + 64 * mb + 16 * wq + 8 * e + px;
        const int wr = L / kC0XW, wc = L - wr * kC0XW;
        if (wc == 0 || wr > 2 * kC0Tile + 2) continue;  // (wr, wc in [1, 18])
        const int hy = hy0 + wr, hx = hx0 + wc;
        const bool inside = hy >= 0 && hy < H2 && hx >= 0 && hx < W2;
        const uint32_t cell = (uint32_t)(((wr - 1) >> 1) * (kC0Tile + 1) + ((wc - 1) >> 1));
        const uint32_t base = c00 + (((wr - 1) & 1) ? p.c00_kb1 : 0u) + 4u * (lane & 3);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float a0 = acc0[mb][4 * j + 2 * e] + sh0[j].x, a1 = acc0[mb][4 * j + 2 * e + 1] + sh0[j].y;
          const uint32_t v = inside ? Pack2<T>::pack(fmaxf(a0, 0.2f * a0), fmaxf(a1, 0.2f * a1)) : 0u;
          st_shared_u32(base + swz_off(cell, (uint32_t)(((wc - 1) & 1) * 4 + j), 128u), v);
        }
      }
    fence_proxy_async();  // the generic-proxy window writes before the tensor cores read them
    named_bar_sync(1 + g, 128);

    // ---- conv0.1 on that window: one m64 row block, 9 runs of 2 K=16 steps
    wgmma_fence();
#pragma unroll
    for (int r = 0; r < 9; ++r) {
      const uint4 d = p.mma1[r];
      const uint64_t a64 = ((uint64_t)d.y << 32) | (uint64_t)(c00_lo + d.x);
      const uint64_t b64 = ((uint64_t)p.b_hi << 32) | (uint64_t)(b1_lo + d.z);
#pragma unroll
      for (int i = 0; i < 2; ++i) wgmma_ss<64, T>(acc1, a64 + 2u * i, b64 + 2u * i, (r | i) ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc1);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      acc1[4 * j] += sh1[j].x;
      acc1[4 * j + 1] += sh1[j].y;
      acc1[4 * j + 2] += sh1[j].x;
      acc1[4 * j + 3] += sh1[j].y;
    }
    if (leader) bulk_wait_read<0>();  // the previous tile's store has read the staging tile
    named_bar_sync(1 + g, 128);      // (also: every warp's conv0.1 MMAs are done before the next tile rewrites the window)
    stage_rows<64, T>(acc1, out_smem, kC0OutBytes, 2 * wq, lane, 0.2f);
    fence_proxy_async();
    named_bar_sync(1 + g, 128);
    if (leader) {
      tma_store_4d(&p.tm_out, out_smem, 0, kC0Tile * it.tx, kC0Tile * it.ty, it.b);
      bulk_commit();
    }
  }
  if (leader) bulk_wait<0>();
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
  p.wstream = L.wstream;
  if (L.ktotal16 > kMaxK16) return 0;
  // n_cta = the wgmma N: whole 8-row swizzle atoms of B, and a multiple of 16 with an instantiated kernel (<= 96: two
  // 64-row accumulators of n_cta fp32 columns per thread)
  // (streamed weights, whose shift is read per tile instead: up to 128)
  if (p.nkb > kMaxKBlocks || L.n_cta > (L.wstream ? 128 : 96) || (L.n_cta & 15) || L.n_cta < 16) return 0;
  if (L.wstream && (L.ktotal16 & 3)) return 0;
  uint32_t off = 0;
  p.tx_bytes = 0;
  for (int kb = 0; kb < p.nkb; ++kb) {
    const bool tail = (kb == p.nkb - 1) && (L.cin & 63);
    const uint32_t bytes = (uint32_t)L.halo_w * (uint32_t)L.halo_h * (tail ? 64u : 128u);
    p.kb_off[kb] = off;
    off += align_up(bytes, 1024);
    p.tx_bytes += bytes;
  }
  p.stage_bytes = off;
  {
    // wgmma descriptor words per K=16 step (ptx.cuh): start>>4 [0,14) | LBO [16,30) ; SBO>>4 [32,46) | layout [62,64)
    // (1 = SWIZZLE_128B, 2 = SWIZZLE_64B); base_offset stays 0.
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
    // (streamed weights: one entry per step, issue_wslot)
    int run_len = 1;
    for (int len : {4, 2}) {
      if (L.wstream) break;
      bool ok = (L.ktotal16 % len) == 0;
      for (int r = 0; ok && r < L.ktotal16; r += len)
        for (int i = 1; i < len; ++i)
          ok = ok && step[r + i].x == step[r].x + 2u * i && step[r + i].y == step[r].y &&
               step[r + i].z == step[r].z + 2u * i;
      if (ok) {
        run_len = len;
        break;
      }
    }
    p.run_len = run_len;
    p.nruns = L.ktotal16 / run_len;
    for (int r = 0; r < p.nruns; ++r) p.mma[r] = step[r * run_len];
  }
  p.b_hi = (1024u >> 4) | kDescSw128;  // B: SBO = 8 rows x 128 B, SWIZZLE_128B
  p.off_w = align_up(kCtrlBytes, 1024);
  // 16-bit NHWC outputs leave through TMA tensor stores from one staging tile per MMA warpgroup (128 cells x n_cta
  // channels, 1024-aligned store boxes).  A dedicated region rather than the consumed window stage: the stage is free
  // for the next fill as soon as the residual is read.  The staging costs window stages; a resident-weight layer left
  // with fewer than kMinStagedStages keeps direct stores (on H100 at 1080p conv0.1 at c = 96 / 192 lost more than the
  // stores gained).  lastconv's fp32 planes and the space-to-depth / patch forms always store directly.
  constexpr int kMinStagedStages = 3;
  const uint32_t staged_out =
      (L.epi_mode != EPI_LASTCONV && L.out_s2d == 0) ? (uint32_t)(kTileH * kTileW) * L.n_cta * 2u : 0u;
  auto fit = [&](uint32_t out_stage) {
    p.out_stage_bytes = out_stage;
    p.off_out = align_up(p.off_w + p.w_bytes, 1024);
    p.off_a = p.off_out + kMmaGroups * out_stage;
    for (int s = kMaxStages; s >= 1; --s)
      if (p.off_a + (uint32_t)s * p.stage_bytes <= (uint32_t)kSmemLimit) return s;
    return 0;
  };
  int stages = 0;
  p.w_groups = (L.ktotal16 + 3) / 4;
  p.w_slot_bytes = (uint32_t)L.n_cta * 128u;
  p.w_slots = 0;
  if (L.wstream) {
    // the weight region holds w_slots slots of four K=16 steps.  Preference: the staged stores (both warpgroups run
    // their epilogues at once, the tensor cores idle meanwhile), then 4 window stages (the next pass's windows load
    // during this one) down to the 2 the two tiles of a pass need, each with at least 3 weight slots in flight
    constexpr int kMinWSlots = 3;
    for (uint32_t out_stage : {staged_out, 0u})
      for (int s = 4; s >= 2 && p.w_slots == 0; --s) {
        const uint32_t fixed = align_up(kCtrlBytes, 1024) + kMmaGroups * out_stage + (uint32_t)s * p.stage_bytes;
        if (fixed >= (uint32_t)kSmemLimit) continue;
        const int slots = std::min<int>({(int)(((uint32_t)kSmemLimit - fixed) / p.w_slot_bytes), kMaxWSlots, p.w_groups});
        if (slots < std::min(kMinWSlots, p.w_groups)) continue;
        p.w_slots = slots;
        p.w_bytes = (uint32_t)slots * p.w_slot_bytes;  // (resident size for fit(); restored below)
        stages = fit(out_stage);
        p.w_bytes = (uint32_t)p.w_groups * p.w_slot_bytes;
        break;
      }
    if (p.w_slots == 0) return 0;
    p.stages = stages;
    p.smem_bytes = p.off_a + (uint32_t)stages * p.stage_bytes;
    p.cmajor = 0;
    return stages;
  }
  if (staged_out) stages = fit(staged_out);
  if (stages < kMinStagedStages) stages = fit(0u);
  p.stages = stages;
  p.smem_bytes = p.off_a + (uint32_t)stages * p.stage_bytes;  // stage sizes are multiples of 1024
  // Channel-major MMAs (top of this file) need exactly 64 output channels for the M of one wgmma, the whole window
  // held until the epilogue (its residual read) and the staging tile the transposed fragments are stored through.  The
  // shared-memory plan is the same in both orientations.
  p.cmajor = (L.n_cta == 64 && p.out_stage_bytes != 0 && p.nruns == kCmRuns && p.run_len == kCmRunLen) ? 1 : 0;
  return stages;
}

cudaError_t launch_tapconv(const TapConvLayer& L, int op_type, const void* in, void* out, float4* out_flow,
                           float* out_mask, int B, int H, int W, int num_sms, int impl, cudaStream_t st) {
  TapConvParams p{};
  if (tapconv_plan(L, &p) < 1) {
    set_error("tapconv: layer does not fit in shared memory");
    return cudaErrorInvalidConfiguration;
  }
  if (impl == TAPCONV_CELL_MAJOR) p.cmajor = 0;
  bool use_ref = impl == TAPCONV_CHECKER;
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
  if (p.out_stage_bytes) {
    const int bc = store_box_c(L.n_cta);
    const CUtensorMapSwizzle swz = bc == 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                                   : bc == 32 ? CU_TENSOR_MAP_SWIZZLE_64B
                                              : CU_TENSOR_MAP_SWIZZLE_32B;
    if (!make_tmap(&p.tm_out, dt, out, L.n_total, W, H, B, bc, kTileW, kTileH, swz)) return cudaErrorInvalidValue;
  }
  // cps persistent CTAs per output-channel split
  int cps = num_sms / L.nsplit;
  if (cps < 1) cps = 1;
  if (cps > p.ntiles) cps = p.ntiles;
  p.ctas_per_split = cps;
  const int grid = cps * L.nsplit;
  cudaError_t err;  // (per device: set on every launch, it is a cheap driver call)
  auto go = [&](auto kern) -> cudaError_t {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3((unsigned)(p.wstream ? kThreadsWS : kThreads));
    cfg.dynamicSmemBytes = p.smem_bytes;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, p);
  };
  auto pick_n = [&](auto tag, auto lst) -> cudaError_t {
    using T = decltype(tag);
    constexpr bool LA = decltype(lst)::value;
    if (p.wstream) {
      // n_cta = 96 (ResConv c = 96, 192) or 128 (ResConv c = 128, the 4.26 feature conv); lastconv: all 80 columns
      if constexpr (LA) {
        if (L.n_cta == 80) return go(tapconv_kernel<T, true, 80, false, true>);
      } else {
        if (L.n_cta == 96) return go(tapconv_kernel<T, false, 96, false, true>);
        if (L.n_cta == 128) return go(tapconv_kernel<T, false, 128, false, true>);
      }
      set_error("tapconv: streamed weights are instantiated for n_cta = 96 and 128 (lastconv: 80) only");
      return cudaErrorInvalidConfiguration;
    }
    if constexpr (!LA)
      if (p.cmajor) return go(tapconv_kernel<T, false, 64, true, false>);  // (tapconv_plan: n_cta == 64)
    switch (L.n_cta) {  // tapconv_plan admits multiples of 16 up to 96
      case 16: return go(tapconv_kernel<T, LA, 16, false, false>);
      case 32: return go(tapconv_kernel<T, LA, 32, false, false>);
      case 48: return go(tapconv_kernel<T, LA, 48, false, false>);
      case 64: return go(tapconv_kernel<T, LA, 64, false, false>);
      case 80: return go(tapconv_kernel<T, LA, 80, false, false>);
      default: return go(tapconv_kernel<T, LA, 96, false, false>);
    }
  };
  auto pick = [&](auto tag) -> cudaError_t {
    return L.epi_mode == EPI_LASTCONV ? pick_n(tag, std::true_type{}) : pick_n(tag, std::false_type{});
  };
  err = (op_type == OP_BF16) ? pick(__nv_bfloat16{}) : pick(__half{});
  if (err != cudaSuccess) return err;
  return cudaGetLastError();
#endif  // VFI_HOST_EMU
}

int conv0_fused_plan(const TapConvLayer& L0, const TapConvLayer& L1, int op_type, int* smem_bytes, int* regs,
                     int* local_bytes) {
  Conv0Params p{};
  if (!conv0_fused_layout(L0, L1, &p)) return 0;
  int r = 0, lb = 0;
#ifndef VFI_HOST_EMU
  cudaFuncAttributes fa{};
  const void* kern = op_type == OP_BF16 ? (const void*)conv0_fused_kernel<__nv_bfloat16> : (const void*)conv0_fused_kernel<__half>;
  if ((regs || local_bytes) && cudaFuncGetAttributes(&fa, kern) == cudaSuccess) {
    r = fa.numRegs;
    lb = (int)fa.localSizeBytes;
  }
#else
  (void)op_type;
#endif
  if (smem_bytes) *smem_bytes = (int)p.smem_bytes;
  if (regs) *regs = r;
  if (local_bytes) *local_bytes = lb;
  return kMmaGroups;  // x window stages: one per MMA warpgroup
}

cudaError_t launch_conv0_fused(const TapConvLayer& L0, const TapConvLayer& L1, int op_type, const void* x, void* c00,
                               void* out, int B, int H, int W, int num_sms, cudaStream_t st) {
  Conv0Params p{};
  if (!conv0_fused_layout(L0, L1, &p)) {
    set_error("conv0 fused: the layers are not a 64-channel arch-4.6 conv0.0 / conv0.1 pair");
    return cudaErrorInvalidConfiguration;
  }
  if (B < 1 || H < 2 || W < 2 || ((H | W) & 1)) {
    set_error("conv0 fused: the conv0.0 grid needs even H and W");
    return cudaErrorInvalidValue;
  }
#ifdef VFI_HOST_EMU
  // the host emulation has only the checker kernel: the two launches, through c00
  if (!c00) return cudaErrorInvalidValue;
  const cudaError_t e = launch_tapconv(L0, op_type, x, c00, nullptr, nullptr, B, H, W, num_sms, TAPCONV_CHECKER, st);
  if (e != cudaSuccess) return e;
  return launch_tapconv(L1, op_type, c00, out, nullptr, nullptr, B, H / 2, W / 2, num_sms, TAPCONV_CHECKER, st);
#else
  (void)c00;
  const CUtensorMapDataType dt = (op_type == OP_BF16) ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  p.H4 = H / 2;
  p.W4 = W / 2;
  if (!make_tmap(&p.tm_x, dt, x, 64, W, H, B, 64, kC0XW, kC0XW, CU_TENSOR_MAP_SWIZZLE_128B) ||
      !make_tmap(&p.tm_out, dt, out, 64, p.W4, p.H4, B, 64, kC0Tile, kC0Tile, CU_TENSOR_MAP_SWIZZLE_128B))
    return cudaErrorInvalidValue;
  p.w0 = L0.w;
  p.w1 = L1.w;
  p.shift0 = L0.shift;
  p.shift1 = L1.shift;
  p.B = B;
  p.tiles_y = (p.H4 + kC0Tile - 1) / kC0Tile;
  p.tiles_x = (p.W4 + kC0Tile - 1) / kC0Tile;
  p.ntiles = B * p.tiles_y * p.tiles_x;
  p.ctas = std::max(1, std::min(num_sms, p.ntiles));
  auto kern = (op_type == OP_BF16) ? conv0_fused_kernel<__nv_bfloat16> : conv0_fused_kernel<__half>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
  if (e != cudaSuccess) return e;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)p.ctas);
  cfg.blockDim = dim3((unsigned)kThreads);
  cfg.dynamicSmemBytes = p.smem_bytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  e = cudaLaunchKernelEx(&cfg, kern, p);
  if (e != cudaSuccess) return e;
  return cudaGetLastError();
#endif  // VFI_HOST_EMU
}

}  // namespace vfi
