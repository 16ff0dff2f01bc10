// streamconv: implicit-GEMM convolution with STREAMED weights on the Hopper tensor cores (wgmma / TMA / mbarrier),
// sm_90a only.  The conv kernel of the FILM path (SURVEY.md section 8 row a10), of the Sepconv trunk and of FLAVR, whose
// 3-D convolutions add a temporal tap axis: the A producer walks (temporal tap, k-block) pairs (see src_image).
//
// Replaces the cuDNN / ATen kernels behind film_arch.conv (film_arch.py:784-798: Conv2d(k x k, padding='same')
// [+ LeakyReLU(0.2)], k = 1, 2, 3) for every layer of
//   SubTreeExtractor (film_arch.py:91-121), FlowEstimator (:515-543) and Fusion (:222-296)
// whose input has >= 64 channels: 64 ... 2442 input channels, 16 ... 512 output channels.
//
// Why a second conv kernel: tapconv.cu keeps a layer's whole weight slice resident in shared memory (RIFE: <= 110 KB
// per CTA).  FILM's layers have up to 9 x 2442 x 512 weights (22 MB), so here BOTH operands stream:
//   A  the input window of a tile (tile + halo) for ONE 64-channel k-block, dropped into shared memory by TMA as rows of
//      128 B (SWIZZLE_128B) - the layout of one k-block of tapconv's staged window: every filter tap is a descriptor
//      START ADDRESS into the window ((dy*halo_w + dx) * 128 B, 8-row-group stride SBO = halo_w * 128 B), a K=16 step a
//      32-byte shift.  One CTA pass covers mt = 2 tiles of 16 x 8 output pixels, one per MMA warpgroup, so a weight
//      slice read from L2 feeds 2 x 128 rows;
//   B  the weights of one (k-block, tap): [n_cta rows][64 channels = 128 B, 16-byte chunks XOR (n & 7)] = the
//      SWIZZLE_128B K-major B operand bit for bit, packed that way on the host, one cp.async.bulk per slot.
// A layer may read its input channels from TWO tensors (k-blocks [0, nkb0) from source 0, the rest from source 1):
// torch.cat along channels (film_arch.py:541, :292, :781) never materialises.  Channel counts are padded to multiples of
// 64 in HBM (zero weights for the padding), outputs go to any channel slice of a wider NHWC tensor.
//
// Warp roles (320 threads, 1 persistent CTA per SM):
//   warpgroups 0, 1 : warpgroup t multiplies tile t of the pass (two m64 row blocks, accumulators in registers) and
//                     runs its epilogue: + bias -> LeakyReLU / identity (ext: PReLU, + residual) -> 16-bit -> stores
//   warp 8          : one elected lane: A producer (one 4-D TMA per tile and k-block)
//   warp 9          : one elected lane: B producer (one bulk copy per (k-block, tap))
// Pipelines: A ring (2-4 slots, full = TMA bytes, empty = both warpgroups after the k-block's last tap), B ring (3-8
// slots, full = bulk-copy bytes, empty = both warpgroups after the tap's MMAs have completed).  Every wait is bounded
// (ptx.cuh mbar_wait) and traps.
#include <cstring>
#include <type_traits>

#include "ptx.cuh"
#include "vfi_internal.h"

namespace vfi {

namespace {

constexpr int kMaxASlots = 4, kMaxBSlots = 8;
struct SCtrl {
  uint64_t a_full[kMaxASlots];
  uint64_t a_empty[kMaxASlots];
  uint64_t b_full[kMaxBSlots];
  uint64_t b_empty[kMaxBSlots];
};
constexpr uint32_t kSCtrlBytes = 256;
static_assert(sizeof(SCtrl) <= kSCtrlBytes, "control block");
constexpr int kSMmaGroups = 2, kSAWarp = 8, kSBWarp = 9, kSThreads = 128 * kSMmaGroups + 64;
// every warp of both MMA warpgroups arrives on an `empty` barrier once it has waited for the MMAs that read the slot
constexpr uint32_t kSConsumerArrivals = 4 * kSMmaGroups;

struct TileCoord {
  int b, ty, tx;
};
// tile index -> (output image, tile row, tile column); tiles past the end map to image B: nothing is stored
__device__ __forceinline__ TileCoord tile_coord(const StreamConvParams& p, int tile) {
  TileCoord c;
  if (tile >= p.ntiles) {
    c.b = p.B;
    c.ty = 0;
    c.tx = 0;
    return c;
  }
  const int per_img = p.tiles_x * p.tiles_y;
  c.b = tile / per_img;
  const int rem = tile - c.b * per_img;
  c.ty = rem / p.tiles_x;
  c.tx = rem - c.ty * p.tiles_x;
  return c;
}

// input image that temporal tap dt of output image b reads: images are (sample, plane) pairs, b = s * T_out + t_out,
// and the tap reads plane t_out + dt - pad_t of the same sample.  A plane outside [0, T_in) and the images of tiles past
// the end map to image B_in, one past the end of the input tensor: TMA zero-fills it, the checker skips it.
__device__ __forceinline__ int src_image(const StreamConvParams& p, int b, int dt) {
  const int s = b / p.T_out, pl = b - s * p.T_out + dt - p.pad_t;
  return (b >= p.B || pl < 0 || pl >= p.T_in) ? p.B_in : s * p.T_in + pl;
}

__device__ __forceinline__ void ring_next(uint32_t& slot, uint32_t& ph, uint32_t n) {
  if (++slot == n) {
    slot = 0;
    ph ^= 1u;
  }
}

#ifndef VFI_HOST_EMU  // (tests/host_emu runs the schedule on the CPU with the checker kernel below; no wgmma there)
// EPI = 0 is the FILM kernel (bias + LeakyReLU(0.2) / identity).  EPI = 1 adds what the Sepconv trunk needs in the
// epilogue: a PReLU with one learned slope (a > 0 ? a : slope * a, any sign / size of slope) and a residual tensor
// added after it (same layout as the output; it may BE the output: every thread reads its two channels before it
// writes them).  EPI = 2 is IFRNet's (ifrnet.cu): a residual added BEFORE a PReLU with one slope per output channel,
// and the first n_f32 output columns stored as fp32 to a separate tensor (flow, mask and residual columns are never
// rounded to 16 bits).
template <typename T, int EPI, int N>
__global__ void __launch_bounds__(kSThreads, 1) streamconv_kernel(const __grid_constant__ StreamConvParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  asm volatile("griddepcontrol.launch_dependents;");  // see tapconv.cu: programmatic dependent launch
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // the k-th pass of this CTA is pass0 + k * pass_stride; passes past the end have no valid tile (zero-filled A, no stores)
  const int split = blockIdx.x % p.nsplit;
  const int first = blockIdx.x / p.nsplit;
  if (first >= p.ctas_per_split) return;
  const int my_passes = (p.npasses - first + p.ctas_per_split - 1) / p.ctas_per_split;
  const int pass0 = first;
  const int pass_stride = p.ctas_per_split;
  const int mt = p.mt;

  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bar_afull = smem_base + offsetof(SCtrl, a_full);
  const uint32_t bar_aempty = smem_base + offsetof(SCtrl, a_empty);
  const uint32_t bar_bfull = smem_base + offsetof(SCtrl, b_full);
  const uint32_t bar_bempty = smem_base + offsetof(SCtrl, b_empty);
  const uint32_t a_smem = smem_base + p.off_a;
  const uint32_t b_smem = smem_base + p.off_b;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.a_slots; ++s) {
      mbar_init(bar_afull + 8 * s, 1);  // producer's arrive.expect_tx (+ TMA bytes)
      mbar_init(bar_aempty + 8 * s, kSConsumerArrivals);
    }
    for (int s = 0; s < p.b_slots; ++s) {
      mbar_init(bar_bfull + 8 * s, 1);
      mbar_init(bar_bempty + 8 * s, kSConsumerArrivals);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == kSAWarp) {
    // ======================================================= A producer
    if (lane == 0) {
      asm volatile("griddepcontrol.wait;" ::: "memory");  // the input is the previous kernels' output
      uint32_t slot = 0, ph = 0;
      for (int k = 0; k < my_passes; ++k) {
        const int pass = pass0 + k * pass_stride;
        TileCoord tc[2];
        tc[0] = tile_coord(p, pass * mt);
        tc[1] = tile_coord(p, pass * mt + 1);
        for (int j = 0; j < p.kt * p.nkb; ++j) {  // (temporal tap, k-block), the order of the packed weights
          const int dt = j / p.nkb, kb = j - dt * p.nkb;
          mbar_wait(bar_aempty + 8 * slot, ph ^ 1u);
          mbar_arrive_expect_tx(bar_afull + 8 * slot, (uint32_t)mt * p.a_tx_bytes);
          const bool s0 = kb < p.nkb0;
          const void* tm = s0 ? &p.tm[0] : &p.tm[1];
          const int c0 = (s0 ? kb : kb - p.nkb0) * 64;
          for (int t = 0; t < mt; ++t)
            tma_load_4d(a_smem + slot * p.a_slot_bytes + (uint32_t)t * p.a_win_bytes, tm, bar_afull + 8 * slot, c0,
                        tc[t].tx * kTileW + p.halo_x0, tc[t].ty * kTileH + p.halo_y0, src_image(p, tc[t].b, dt));
          ring_next(slot, ph, (uint32_t)p.a_slots);
        }
      }
    }
    return;
  }
  if (warp == kSBWarp) {
    // ======================================================= B producer (weights never depend on a previous kernel)
    if (lane == 0) {
      const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(p.w) + (size_t)split * p.w_split_bytes;
      uint32_t slot = 0, ph = 0;
      const int per_pass = p.kt * p.nkb * p.ntaps;
      for (int k = 0; k < my_passes; ++k) {
        for (int j = 0; j < per_pass; ++j) {
          mbar_wait(bar_bempty + 8 * slot, ph ^ 1u);
          mbar_arrive_expect_tx(bar_bfull + 8 * slot, p.b_slot_bytes);
          bulk_g2s(b_smem + slot * p.b_slot_bytes, wsrc + (size_t)j * p.b_slot_bytes, p.b_slot_bytes, bar_bfull + 8 * slot);
          ring_next(slot, ph, (uint32_t)p.b_slots);
        }
      }
    }
    return;
  }

  // ========================================================= MMA + epilogue warpgroups (warpgroup t = tile t of a pass)
  const int t = warp >> 2;
  const int wq = warp & 3;
  asm volatile("griddepcontrol.wait;" ::: "memory");  // our stores may overwrite what the previous kernel still reads
  const uint32_t a_lo0 = (1u << 16) | (a_smem >> 4);   // LBO(=1) | start address, 16-byte units
  const uint32_t b_lo0 = (1u << 16) | (b_smem >> 4);
  const uint32_t b_hi = (1024u >> 4) | kDescSw128;     // SBO = 8 rows x 128 B, SWIZZLE_128B
  const uint32_t a_hi = p.a_hi;                        // SBO = halo_w x 128 B, SWIZZLE_128B
  const uint32_t half_off = 8u * (a_hi & 0x3fffu);      // rows 64..127 of the tile: 8 tile rows further down
  const uint32_t a_slot_u = p.a_slot_bytes >> 4, a_win_u = p.a_win_bytes >> 4, b_slot_u = p.b_slot_bytes >> 4;
  const int n0 = split * p.n_cta;
  const float slope = p.act ? 0.2f : 1.f;  // max(a, slope * a): LeakyReLU(0.2) or identity
  const int px = lane >> 2, c2 = 2 * (lane & 3);
  uint32_t aslot = 0, aph = 0, bslot = 0, bph = 0;
  float acc[2][N / 2];
  for (int k = 0; k < my_passes; ++k) {
    // MMAs of one (k-block, tap) form one wgmma group; the slot of the previous group is released once it completes
    uint32_t prev_b = 0, prev_a = 0;
    bool prev_last_tap = false, have_prev = false;
    for (int kb = 0; kb < p.kt * p.nkb; ++kb) {
      mbar_wait(bar_afull + 8 * aslot, aph);
      for (int tap = 0; tap < p.ntaps; ++tap) {
        mbar_wait(bar_bfull + 8 * bslot, bph);
        wgmma_fence();
        const uint32_t a_lo = a_lo0 + aslot * a_slot_u + (uint32_t)t * a_win_u + p.tap_off[tap];
        const uint32_t b_lo = b_lo0 + bslot * b_slot_u;
        const uint32_t first_mma = (kb | tap) ? 1u : 0u;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          uint64_t a64 = ((uint64_t)a_hi << 32) | (uint64_t)(a_lo + (uint32_t)h * half_off);
          uint64_t b64 = ((uint64_t)b_hi << 32) | (uint64_t)b_lo;
#pragma unroll
          for (int i = 0; i < 4; ++i) {  // 64 channels = four K=16 steps, +32 B each
            wgmma_ss<N, T>(acc[h], a64, b64, i ? 1u : first_mma);
            a64 += 2;
            b64 += 2;
          }
        }
        wgmma_commit();
        if (have_prev) {
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(bar_bempty + 8 * prev_b);
            if (prev_last_tap) mbar_arrive(bar_aempty + 8 * prev_a);
          }
        }
        have_prev = true;
        prev_b = bslot;
        prev_a = aslot;
        prev_last_tap = (tap == p.ntaps - 1);
        ring_next(bslot, bph, (uint32_t)p.b_slots);
      }
      ring_next(aslot, aph, (uint32_t)p.a_slots);
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(bar_bempty + 8 * prev_b);
      mbar_arrive(bar_aempty + 8 * prev_a);
    }
    acc_fence(acc[0]);
    acc_fence(acc[1]);

    // ---- epilogue: d[h][4 j + 2 e + c] = tile row 8 h + 2 wq + e, column 8 j + c2 + c
    const TileCoord tc = tile_coord(p, (pass0 + k * pass_stride) * mt + t);
    if (tc.b >= p.B) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int gy = tc.ty * kTileH + 8 * h + 2 * wq + e, gx = tc.tx * kTileW + px;
        if (gy >= p.H || gx >= p.W) continue;
        const size_t opix = (((size_t)tc.b * p.H + gy) * p.W + gx) * (size_t)p.out_pitch + (size_t)n0;
        T* orow = reinterpret_cast<T*>(p.out) + opix;
        const T* rrow = reinterpret_cast<const T*>(p.res) + opix;  // EPI 1, 2 only
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
          const int n = 8 * j + c2;
          const float2 sh = *reinterpret_cast<const float2*>(p.shift + n0 + n);
          float a0 = acc[h][4 * j + 2 * e] + sh.x, a1 = acc[h][4 * j + 2 * e + 1] + sh.y;
          uint32_t o;
          if constexpr (EPI == 2) {
            if (p.res != nullptr) {
              const float2 rf = Pack2<T>::unpack(*reinterpret_cast<const uint32_t*>(rrow + n));
              a0 += rf.x;
              a1 += rf.y;
            }
            const float2 sl = *reinterpret_cast<const float2*>(p.slopes + n0 + n);
            a0 = a0 > 0.f ? a0 : sl.x * a0;
            a1 = a1 > 0.f ? a1 : sl.y * a1;
            // the fp32 columns lie in the first 8 of split 0 (launch_streamconv checks n_f32 <= 8)
            if (j == 0 && n0 + n < p.n_f32) {
              const size_t fpix = (((size_t)tc.b * p.H + gy) * p.W + gx) * (size_t)p.f32_pitch;
              *reinterpret_cast<float2*>(p.out_f32 + fpix + n) = make_float2(a0, a1);
              continue;
            }
            o = Pack2<T>::pack(a0, a1);
          } else if constexpr (EPI == 1) {
            a0 = a0 > 0.f ? a0 : p.slope * a0;
            a1 = a1 > 0.f ? a1 : p.slope * a1;
            if (p.res != nullptr) {
              const float2 rf = Pack2<T>::unpack(*reinterpret_cast<const uint32_t*>(rrow + n));
              a0 += rf.x;
              a1 += rf.y;
            }
            o = Pack2<T>::pack(a0, a1);
          } else {
            o = Pack2<T>::pack(fmaxf(a0, slope * a0), fmaxf(a1, slope * a1));
          }
          *reinterpret_cast<uint32_t*>(orow + n) = o;
        }
      }
  }
}

#endif  // VFI_HOST_EMU

// ---------------------------------------------------------------------------------------------
// CUDA-core checker with the SAME parameters and packed weights: one thread per (pixel, n).
// Test infrastructure for the tensor-core kernel (debug entry points only; never on the product path).
// ---------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float sc_ld(const T* p);
template <>
__device__ __forceinline__ float sc_ld<__half>(const __half* p) { return __half2float(*p); }
template <>
__device__ __forceinline__ float sc_ld<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }

template <typename T>
__device__ __forceinline__ T sc_cvt(float v);
template <>
__device__ __forceinline__ __half sc_cvt<__half>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 sc_cvt<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <typename T>
__global__ void streamconv_ref_kernel(const __grid_constant__ StreamConvParams p) {
  const size_t total = (size_t)p.B * p.H * p.W * p.n_total;
  for (size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(id % p.n_total);
    size_t cell = id / p.n_total;
    const int gx = (int)(cell % p.W);
    cell /= p.W;
    const int gy = (int)(cell % p.H);
    const int b = (int)(cell / p.H);
    const int split = n / p.n_cta, nl = n - split * p.n_cta;
    const T* w = reinterpret_cast<const T*>(reinterpret_cast<const uint8_t*>(p.w) + (size_t)split * p.w_split_bytes);
    float acc = 0.f;
    for (int dt = 0; dt < p.kt; ++dt) {
      const int img = src_image(p, b, dt);
      if (img >= p.B_in) continue;
      for (int kb = 0; kb < p.nkb; ++kb) {
        const bool s0 = kb < p.nkb0;
        const T* src = reinterpret_cast<const T*>(s0 ? p.src[0] : p.src[1]);
        const int pitch = s0 ? p.src_pitch[0] : p.src_pitch[1];
        const int c0 = (s0 ? kb : kb - p.nkb0) * 64;
        for (int tap = 0; tap < p.ntaps; ++tap) {
          const int y = gy + p.halo_y0 + tap / p.ksize, x = gx + p.halo_x0 + tap % p.ksize;
          if (y < 0 || y >= p.H || x < 0 || x >= p.W) continue;
          const T* px = src + (((size_t)img * p.H + y) * p.W + x) * (size_t)pitch + c0;
          const T* wr = w + ((size_t)((dt * p.nkb + kb) * p.ntaps + tap) * p.n_cta + nl) * 64;
          for (int c = 0; c < 64; ++c) {
            const int chunk = c >> 3;
            acc = fmaf(sc_ld<T>(px + c), sc_ld<T>(wr + ((chunk ^ (nl & 7)) * 8 + (c & 7))), acc);
          }
        }
      }
    }
    float v = acc + p.shift[n];
    const size_t oidx = (((size_t)b * p.H + gy) * p.W + gx) * (size_t)p.out_pitch + n;
    if (p.ext == 2) {
      if (p.res != nullptr) v += sc_ld<T>(reinterpret_cast<const T*>(p.res) + oidx);
      v = v > 0.f ? v : p.slopes[n] * v;
      if (n < p.n_f32) {
        p.out_f32[(((size_t)b * p.H + gy) * p.W + gx) * (size_t)p.f32_pitch + n] = v;
        continue;
      }
    } else if (p.ext) {
      v = v > 0.f ? v : p.slope * v;
      if (p.res != nullptr) v += sc_ld<T>(reinterpret_cast<const T*>(p.res) + oidx);
    } else if (p.act) {
      v = lrelu02(v);
    }
    T* o = reinterpret_cast<T*>(p.out) + oidx;
    *o = sc_cvt<T>(v);
  }
}

#ifndef VFI_HOST_EMU
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// a channel slice [C of pitch] of an NHWC tensor as a 4-D tensor {C, W, H, B}, box {64, box_w, box_h, 1}, SWIZZLE_128B
bool make_slice_tmap(CUtensorMap* tm, CUtensorMapDataType dt, const void* base, int C, int pitch, int W, int H, int B,
                     int box_w, int box_h) {
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
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  const cuuint64_t strides[3] = {(cuuint64_t)pitch * 2, (cuuint64_t)W * pitch * 2, (cuuint64_t)H * W * pitch * 2};
  const cuuint32_t box[4] = {64u, (cuuint32_t)box_w, (cuuint32_t)box_h, 1u};
  const cuuint32_t es[4] = {1, 1, 1, 1};
  const CUresult r = fn(tm, dt, 4, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
    return false;
  }
  return true;
}

#endif  // VFI_HOST_EMU

uint32_t sc_align_up(uint32_t v, uint32_t a) { return (v + a - 1) / a * a; }

}  // namespace

// Tile / pipeline plan of a layer.  Returns false when the layer cannot run (bad channel counts).
bool streamconv_plan(const StreamConvLayer& L, StreamConvParams* pp) {
  StreamConvParams& p = *pp;
  if (L.ksize < 1 || L.ksize > 3 || L.c0 % 64 || L.c1 % 64 || L.c0 < 64 || L.n_total % 16 || L.n_total < 16) return false;
  if (L.kt < 1 || L.kt > 4 || L.pad_t < 0 || L.T_in < 1 || L.T_out < 1) return false;
  p.ksize = L.ksize;
  p.ntaps = L.ksize * L.ksize;
  // padding='same': (k-1)/2 before, the rest after (film_arch.py:789); L.pad_before >= 0 overrides it (Sepconv's stride-2
  // convs run as 2x2 convs over a space-to-depth input with their one padding row / column BEFORE); L.pad_before_x >= 0
  // sets the columns apart from the rows (the phases of a transposed conv, flavr.cu)
  p.halo_y0 = -(L.pad_before >= 0 ? L.pad_before : (L.ksize - 1) / 2);
  p.halo_x0 = L.pad_before_x >= 0 ? -L.pad_before_x : p.halo_y0;
  p.kt = L.kt;
  p.pad_t = L.pad_t;
  p.T_in = L.T_in;
  p.T_out = L.T_out;
  p.halo_h = kTileH + L.ksize - 1;
  p.halo_w = kTileW + L.ksize - 1;
  p.nkb0 = L.c0 / 64;
  p.nkb = (L.c0 + L.c1) / 64;
  p.n_total = L.n_total;
  p.act = L.act;
  // output channels per CTA (the wgmma N): the whole layer up to 128, else 128-wide splits (n_total = 256, 512)
  int n_cta = L.n_total < 128 ? L.n_total : 128;
  while (L.n_total % n_cta) n_cta -= 16;
  p.n_cta = n_cta;
  p.nsplit = L.n_total / n_cta;
  p.mt = kSMmaGroups;  // one tile per MMA warpgroup
  p.b_slot_bytes = (uint32_t)n_cta * 128u;
  p.w_split_bytes = (size_t)p.kt * p.nkb * p.ntaps * p.b_slot_bytes;
  p.a_tx_bytes = (uint32_t)p.halo_w * (uint32_t)p.halo_h * 128u;
  p.a_win_bytes = sc_align_up(p.a_tx_bytes, 1024);
  p.a_slot_bytes = (uint32_t)p.mt * p.a_win_bytes;
  p.off_b = sc_align_up(kSCtrlBytes, 1024);
  // shared memory: at least 2 window slots and 3 weight slots; then a third window slot if 4 weight slots still fit;
  // the rest goes to weight slots (a window slot lasts ntaps x mt x 4 MMAs, a weight slot mt x 4)
  int a_slots = 2;
  auto fits = [&](int as, int bs) {
    return p.off_b + (uint32_t)bs * p.b_slot_bytes + (uint32_t)as * p.a_slot_bytes <= (uint32_t)kSmemLimit;
  };
  if (!fits(2, 3)) return false;
  if (fits(3, 4)) a_slots = 3;
  int b_slots = 3;
  while (b_slots < kMaxBSlots && fits(a_slots, b_slots + 1)) ++b_slots;
  p.a_slots = a_slots;
  p.b_slots = b_slots;
  p.off_a = p.off_b + (uint32_t)b_slots * p.b_slot_bytes;  // multiples of 2048: 1024-aligned
  p.smem_bytes = p.off_a + (uint32_t)a_slots * p.a_slot_bytes;
  p.a_hi = (((uint32_t)p.halo_w * 128u) >> 4) | kDescSw128;
  for (int tap = 0; tap < p.ntaps; ++tap)
    p.tap_off[tap] = ((uint32_t)((tap / L.ksize) * p.halo_w + (tap % L.ksize)) * 128u) >> 4;
  return true;
}

// 16-bit operand element of a weight (host)
static uint16_t to_op(float v, int op_type) {
  uint16_t u;
  if (op_type == OP_BF16) {
    __nv_bfloat16 h = __float2bfloat16_rn(v);
    std::memcpy(&u, &h, 2);
  } else {
    __half h = __float2half_rn(v);
    std::memcpy(&u, &h, 2);
  }
  return u;
}

// Host-only operand packer (flavr.cu): wfun(output column n, temporal tap dt, tap = ky * k + kx, padded input channel) ->
// weight; layout [split][dt][k-block][tap][n_cta rows][64 channels = 128 B, 16-byte chunks XOR (row & 7)] = what one B
// slot receives, in the order the B producer streams them.
bool pack_streamconv3d(const StreamConvLayer& L, int op_type, const std::function<float(int, int, int, int)>& wfun,
                       std::vector<uint16_t>* out, StreamConvParams* plan) {
  StreamConvParams& p = *plan;
  p = StreamConvParams{};
  if (!streamconv_plan(L, &p)) return false;
  const int ntaps = L.ksize * L.ksize;
  const size_t per_split = (size_t)L.kt * p.nkb * ntaps * p.n_cta * 64;
  std::vector<uint16_t>& pk = *out;
  pk.assign((size_t)p.nsplit * per_split, 0);
  for (int sp = 0; sp < p.nsplit; ++sp)
    for (int dt = 0; dt < L.kt; ++dt)
      for (int kb = 0; kb < p.nkb; ++kb)
        for (int tap = 0; tap < ntaps; ++tap)
          for (int nl = 0; nl < p.n_cta; ++nl) {
            uint16_t* row = &pk[sp * per_split + ((size_t)((dt * p.nkb + kb) * ntaps + tap) * p.n_cta + nl) * 64];
            for (int c = 0; c < 64; ++c) {
              const float val = wfun(sp * p.n_cta + nl, dt, tap, kb * 64 + c);
              if (val != 0.f) row[(((c >> 3) ^ (nl & 7)) * 8) + (c & 7)] = to_op(val, op_type);
            }
          }
  return true;
}

// 2-D form (film.cu, sepconv.cu): wfun(output column n, tap = ky * k + kx, padded input channel) -> weight
bool pack_streamconv(const StreamConvLayer& L, int op_type, const std::function<float(int, int, int)>& wfun,
                     std::vector<uint16_t>* out, StreamConvParams* plan) {
  return pack_streamconv3d(L, op_type, [&](int n, int, int tap, int j) { return wfun(n, tap, j); }, out, plan);
}

cudaError_t launch_streamconv(const StreamConvLayer& L, int op_type, const void* src0, int pitch0, const void* src1,
                              int pitch1, void* out, int out_pitch, int B, int H, int W, int num_sms, bool use_ref,
                              cudaStream_t st, const void* res, float* out_f32, int f32_pitch) {
  StreamConvParams p{};
  if (!streamconv_plan(L, &p)) {
    set_error("streamconv: unsupported layer shape");
    return cudaErrorInvalidConfiguration;
  }
  if ((pitch0 & 7) || (L.c1 && (pitch1 & 7)) || (out_pitch & 15) || ((uintptr_t)out & 31) || ((uintptr_t)src0 & 15) ||
      ((uintptr_t)src1 & 15)) {
    set_error("streamconv: tensor slices must be 16-byte (inputs) / 32-byte (output) aligned");
    return cudaErrorInvalidValue;
  }
  p.src[0] = src0;
  p.src[1] = L.c1 ? src1 : src0;
  p.src_pitch[0] = pitch0;
  p.src_pitch[1] = L.c1 ? pitch1 : pitch0;
  p.out = out;
  p.out_pitch = out_pitch;
  p.ext = L.ext;
  p.slope = L.slope;
  p.res = L.ext ? res : nullptr;
  if (res && !L.ext) {
    set_error("streamconv: a residual needs an ext layer");
    return cudaErrorInvalidValue;
  }
  if ((uintptr_t)res & 31) {
    set_error("streamconv: residual slice must be 32-byte aligned");
    return cudaErrorInvalidValue;
  }
  if (L.ext == 2 && (!L.slopes || (L.n_f32 & 1) || L.n_f32 > 8 ||
                     (L.n_f32 && (!out_f32 || ((uintptr_t)out_f32 & 7) || (f32_pitch & 1) || f32_pitch < L.n_f32)))) {
    set_error("streamconv: an IFRNet epilogue needs its slopes, and an 8-byte aligned fp32 slice for its fp32 columns");
    return cudaErrorInvalidValue;
  }
  p.slopes = L.slopes;
  p.n_f32 = L.ext == 2 ? L.n_f32 : 0;
  p.out_f32 = out_f32;
  p.f32_pitch = f32_pitch;
  p.w = L.w;
  p.shift = L.shift;
  p.B = B * L.T_out;
  p.B_in = B * L.T_in;
  p.H = H;
  p.W = W;
  p.tiles_y = (H + kTileH - 1) / kTileH;
  p.tiles_x = (W + kTileW - 1) / kTileW;
  p.ntiles = p.B * p.tiles_y * p.tiles_x;
  p.npasses = (p.ntiles + p.mt - 1) / p.mt;

  if (use_ref) {
    const size_t total = (size_t)p.B * H * W * L.n_total;
    const int blocks = (int)((total + 255) / 256 < 65535 ? (total + 255) / 256 : 65535);
    if (op_type == OP_BF16)
      VFI_LAUNCH(streamconv_ref_kernel<__nv_bfloat16>, blocks, 256, 0, st, p);
    else
      VFI_LAUNCH(streamconv_ref_kernel<__half>, blocks, 256, 0, st, p);
    return cudaGetLastError();
  }
#ifdef VFI_HOST_EMU
  set_error("streamconv: the host emulation only has the checker kernel");
  return cudaErrorInvalidConfiguration;
#else

  const CUtensorMapDataType dt = (op_type == OP_BF16) ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  if (!make_slice_tmap(&p.tm[0], dt, src0, L.c0, pitch0, W, H, p.B_in, p.halo_w, p.halo_h)) return cudaErrorInvalidValue;
  if (L.c1) {
    if (!make_slice_tmap(&p.tm[1], dt, src1, L.c1, pitch1, W, H, p.B_in, p.halo_w, p.halo_h)) return cudaErrorInvalidValue;
  } else {
    p.tm[1] = p.tm[0];
  }
  int cps = num_sms / p.nsplit;  // persistent CTAs per output-channel split
  if (cps < 1) cps = 1;
  if (cps > p.npasses) cps = p.npasses;
  p.ctas_per_split = cps;
  const int grid = cps * p.nsplit;
  auto go = [&](auto kern) -> cudaError_t {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3((unsigned)kSThreads);
    cfg.dynamicSmemBytes = p.smem_bytes;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, p);
  };
  auto pick_n = [&](auto tag, auto epi) -> cudaError_t {
    using T = decltype(tag);
    constexpr int X = decltype(epi)::value;
    switch (p.n_cta) {  // streamconv_plan: a multiple of 16 up to 128
      case 16: return go(streamconv_kernel<T, X, 16>);
      case 32: return go(streamconv_kernel<T, X, 32>);
      case 48: return go(streamconv_kernel<T, X, 48>);
      case 64: return go(streamconv_kernel<T, X, 64>);
      case 80: return go(streamconv_kernel<T, X, 80>);
      case 96: return go(streamconv_kernel<T, X, 96>);
      case 112: return go(streamconv_kernel<T, X, 112>);
      default: return go(streamconv_kernel<T, X, 128>);
    }
  };
  auto pick = [&](auto tag) -> cudaError_t {
    switch (L.ext) {
      case 0: return pick_n(tag, std::integral_constant<int, 0>{});
      case 1: return pick_n(tag, std::integral_constant<int, 1>{});
      default: return pick_n(tag, std::integral_constant<int, 2>{});
    }
  };
  const cudaError_t err = (op_type == OP_BF16) ? pick(__nv_bfloat16{}) : pick(__half{});
  if (err != cudaSuccess) return err;
  return cudaGetLastError();
#endif  // VFI_HOST_EMU
}

}  // namespace vfi
