// Implicit-GEMM convolution (2-D / 3-D) for sm_90a: TMA-fed, warpgroup MMAs (wgmma) with register accumulators.
//
// Replaces the F.conv2d / F.conv3d call sites of the reference hot path
// (networks/volumetric_avatar/utils.py:661-788 ResBlock, :894-915 Conv2d_ws/Conv3d_ws,
//  decoder.py:77-81,349-356, local_encoder.py:104-108, warp_generator_resnet.py:99-106).
//
// GEMM view:   D[pixel][cout] = sum_{tap, cin} A[pixel + tap][cin] * W[tap][cout][cin]
//   M = 128 output pixels of one (td x th x tw) box of one sample,
//   N = BN output channels, K = taps * Cin walked in chunks of KC channels.
// im2col-free: for every (tap, k-chunk) the A tile is ONE TMA box load of the channels-last activation
//   tensor at the tap-shifted coordinate; out-of-bounds rows/columns are zero-filled by TMA, which is
//   exactly the conv zero padding.  The box lands in shared memory as [pixel][KC] rows with the
//   128B/64B hardware swizzle = the canonical K-major wgmma operand layout.
// Precision: fp32 activations/weights are pre-split into 16-bit planes (hi, lo[, lo2]); each K step issues
//   hi*hi + hi*lo + lo*hi (3 wgmmas per 16 channels; 6 products with three planes) into an fp32 register accumulator.
//   The tensor core accumulates with truncation, so an accumulator only takes a short chunk of MMAs (24 / 48); every chunk
//   is then added to a second set of fp32 registers with round-to-nearest adds.  Plain bf16/tf32 operands, or one long
//   accumulation chain, do not hold the 1e-3 budget.  The decoder's opt-in fast mode takes ONE scaled fp16 plane per operand
//   (a_lo == w_lo == NULL): one wgmma per product, ~2^-11 relative per operand (DESIGN.md section 2).
// Warp roles: warps 0..7 = two consumer warpgroups (64 tile rows each: wgmma issue, chunk promotion, final phase),
//   warps 8..11 = producer warpgroup (warp 8: TMA, one elected lane issues).
// Main loop: stride-1 convolutions load ONE halo A tile per (kernel column, k-chunk) and serve its kh tap rows through
//   descriptor row offsets (A ring + B ring, "row reuse"); other layers load an {A, B} stage per (tap, k-chunk).
// Persistent CTAs walk tiles round-robin.
#include <type_traits>

#include "common.cuh"
#include "wgmma.cuh"

#include <cudaTypedefs.h>
#include <stdlib.h>

namespace emo {

static constexpr int kConsumerWarps = 8;  // two warpgroups
static constexpr int kThreads = kConsumerWarps * 32 + 128;  // + the producer warpgroup (one TMA warp)
static constexpr int kProducerRegs = 40, kConsumerRegs = 232;  // setmaxnreg split: 128 x 40 + 256 x 232 <= 64 Ki registers
static constexpr int kMaxStages = 8;
static constexpr int kMaxAStages = 4;  // row-reuse mode: depth cap of the A (halo tile) ring
static constexpr int kTileM = 128;
static constexpr int kMaxBN = 128;  // N tile cap: each consumer thread holds 2 x BN/2 fp32 accumulators (chunk + sums)

struct ConvKParams {
  int N, Dout, Hout, Wout, Cout;
  int kd, kh, kw, sd, sh, sw, pd, ph, pw;
  int kchunks;
  int tw, th, td;
  int tiles_w, tiles_h, tiles_d;
  int m_tiles, n_tiles;
  int BN;
  int stages;
  int flush;  // k-steps per accumulation chunk
  int ksplit;   // split-K factor: work item = (tile, K part); part `k` writes its partial sums to ws + k * ws_part_elems
  float* ws;    // split-K fp32 workspace [ksplit][N][Dout][Hout][Wout][Cout] (no initial state needed)
  long long ws_part_elems;
  int dbg;    // EMO_CONV_DEBUG builds only (tools/conv_bound_probe.py): 1 skip TMA loads, 2 skip MMAs, 4 skip the residual /
              // post-add loads, 8 skip the output stores, 16 skip the statistics.  Results are garbage; only the timing is of
              // interest.  256 phase stamps, 512 phase clocks (tools/conv_timeline.py).
  const float* bias;
  const float* residual;
  int res_shift;
  int rD, rH, rW;
  int act;
  const float* post_add;
  float* out;
  int out_nchw;
  double* stats;
  int G, cpg;
  // sub-pixel mode (the PS kernels): 3x3 conv over the nearest-x2 upsampling of the input, evaluated on the LOW-resolution
  // planes.  Dout/Hout/Wout above then describe the low-resolution pixel grid the tiles walk; the output tensor is
  // [N][Dout][oH = 2 Hout][oW = 2 Wout][Cout].  The N-tile index carries the output phase: nt = phase * ntc + channel tile,
  // phase = 2 * (row parity) + (column parity); each phase has its own four 2x2 taps (weights [phase * 4 + tap]).
  int oH, oW;
  int ntc;  // channel tiles per phase (= Cout_pad / BN)
  float out_scale;  // fp16 operands (the F16 kernels): 1 / (activation plane scale * weight plane scale)
  // row-reuse mode (stride-1 convolutions with kh > 1 on tiles of one depth slice): the A operand of a (kernel column,
  // k-chunk) group is ONE halo tile of a_rows = tw * (th + kh - 1) pixels serving all kh tap rows; A ring of `sa` halo tiles,
  // B ring of `sb` weight tiles (see the kernel's producer role)
  int yreuse, sa, sb, a_rows;
  // 1: every tile of the launch starts at channel 0 (one channel tile, ntc == 1), so the bias (x 1 / out_scale) is read once
  // per CTA into kMaxBN floats of shared memory above the planned area, instead of from global memory by every tile
  int bias_smem;
};

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

__device__ __forceinline__ void tma_load_5d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// One elected lane of a converged warp: the TMA operands are then provably uniform.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n.reg .pred p;\nelect.sync _|p, 0xffffffff;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// K-major wgmma operand descriptor (sm_90 GMMA matrix descriptor): start >> 4 [0,14), LBO >> 4 [16,30) (unused for swizzled
// K-major tiles), SBO >> 4 [32,46) = pitch of the 8-row swizzle atoms, layout type [62,64) (1 = SWIZZLE_128B, 2 = SWIZZLE_64B).
template <int KC>
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t saddr) {
  constexpr uint64_t row_bytes = KC * 2;          // 128 or 64
  constexpr uint64_t sbo = (8 * row_bytes) >> 4;  // 8-row swizzle atom pitch
  constexpr uint64_t layout = (KC == 64) ? 1ull : 2ull;
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | (1ull << 16) | (sbo << 32) | (layout << 62);
}

// Tile statistics for the fused GroupNorm: the per-(consumer warp, column) slots (filled by the kernel, then a named barrier)
// are summed in a fixed order - warp 0..7, then the columns of a GroupNorm group - and added to the fp64 global sums.
__device__ __forceinline__ void tile_group_stats(const ConvKParams& p, const float* cs, const float* cq, int n, int n0, int BN, int et, int nthreads) {
  const int cpg = p.cpg;
  if (BN % cpg == 0 && (n0 % cpg) == 0) {
    const int ng = BN / cpg;
    for (int g = et; g < ng; g += nthreads) {
      float a = 0.f, b = 0.f;
      for (int q = 0; q < kConsumerWarps; ++q)
        for (int j = 0; j < cpg; ++j) { a += cs[q * kMaxBN + g * cpg + j]; b += cq[q * kMaxBN + g * cpg + j]; }
      const int gi = (n0 / cpg) + g;
      if (gi < p.G) {
        atomicAdd(&p.stats[((long long)n * p.G + gi) * 2], (double)a);
        atomicAdd(&p.stats[((long long)n * p.G + gi) * 2 + 1], (double)b);
      }
    }
  } else {
    for (int j = et; j < BN; j += nthreads) {
      const int c = n0 + j;
      if (c < p.Cout) {
        const int gi = c / cpg;
        float a = 0.f, b = 0.f;
        for (int q = 0; q < kConsumerWarps; ++q) { a += cs[q * kMaxBN + j]; b += cq[q * kMaxBN + j]; }
        atomicAdd(&p.stats[((long long)n * p.G + gi) * 2], (double)a);
        atomicAdd(&p.stats[((long long)n * p.G + gi) * 2 + 1], (double)b);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------------
// Instrumented build only (-DEMO_CONV_DEBUG, tools/conv_timeline.py): per-CTA time stamps (%globaltimer, ns) of the phases of
// the LAST stamped launch: 0 entry, 1 prologue done, 2 / 3 producer first / last issue, 4 first operands landed, 5 last MMA
// chunk of a tile promoted, 6 final-phase stores issued, 7 statistics done, 8 consumer exit (per tile: last tile wins).
#ifdef EMO_CONV_DEBUG
__device__ unsigned long long g_conv_stamps[160 * 16];
__device__ __forceinline__ unsigned long long emo_gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define EMO_STAMP(k, cond) do { if ((p.dbg & 256) && (cond) && blockIdx.x < 160) g_conv_stamps[blockIdx.x * 16 + (k)] = emo_gtime(); } while (0)
// Per-CTA phase clocks (EMO_CONV_DBG bit 512, tools/conv_timeline.py --phases): consumer thread 0 adds the SM clock cycles
// since its previous mark to slot k, over ALL tiles of the launch (the host zeroes them): 0 waiting for operands, 1 issuing
// the main loop and promoting its chunks, 2 final-phase loads (waited for), 3 activation and stores, 4 statistics and
// barriers, 5 tile set-up (prefetch, bias); slot 7 counts the tiles.
__device__ unsigned long long g_conv_phase[160 * 8];
#define EMO_PHASE(k) do { if ((p.dbg & 512) && et == 0 && blockIdx.x < 160) { const long long t_ = clock64(); \
    atomicAdd(&g_conv_phase[blockIdx.x * 8 + (k)], (unsigned long long)(t_ - ph_t)); ph_t = t_; } } while (0)
// EMO_CONV_DBG bits that switch parts of the final phase off: 4 residual / post-add loads, 8 output stores, 16 statistics
#define EMO_DBG(bits) ((p.dbg & (bits)) != 0)
#else
#define EMO_STAMP(k, cond) do { } while (0)
#define EMO_PHASE(k) do { } while (0)
#define EMO_DBG(bits) false
#endif

struct TMaps {
  CUtensorMap a[3];  // activation planes: hi, lo, lo2
  CUtensorMap b[3];  // weight planes
};

// The convolution kernel proper.  The host's instantiation table (kConvKernels) lists the forms that exist:
//   PS = false, F16 = false   the kernel of every ordinary convolution
//   F16 = true                fp16 operand planes (emo_conv_desc.operand_fp16): fp16 wgmma instead of bf16 and a power-of-two
//       rescale of the finished sums
//   PS = true                 sub-pixel form of `nearest x2 -> 3x3 conv` (emo_conv_desc.upconv):
//       the tiles walk the LOW-resolution pixel grid (p.Hout x p.Wout); the N-tile index carries the output phase
//       (nt = phase * p.ntc + channel tile, phase = 2 * row parity + column parity); each phase has four 2x2 taps on the
//       low-resolution planes (weights [phase * 4 + tap]) and its results land on the pixels of that parity of the
//       [p.oH = 2 p.Hout][p.oW = 2 p.Wout] output.
//   PS = true, F16 = true     the sub-pixel form on one fp16 plane
// KC = channels per k-chunk (64 or 32).
// NP = number of 16-bit planes per operand: 1 -> 1 product (fp16 only, ~2^-11 relative per operand), 2 -> 3 products
// (~2^-16 relative with bf16, ~2^-22 with fp16), 3 -> 6 products (~2^-24, fp32-faithful)
// Three warpgroups: warps 0..7 are two consumer warpgroups (warpgroup w issues the wgmmas of tile rows 64 w .. 64 w + 63, promotes its
// accumulation chunks to fp32 registers and runs the final phase of those rows), warp 8 is the TMA producer; setmaxnreg moves
// the registers of the producer warpgroup to the consumers (acc + chunk = 2 x BN/2 fp32 per thread).
// Final phase in registers: bias (as the accumulation's starting value), residual, activation, post-add, float2 stores of the
// wgmma fragment (two rows x two adjacent channels per 8-channel block), GroupNorm statistics by shuffle reduction.
template <int KC, int NP, bool PS, bool F16>
__global__ void __launch_bounds__(kThreads, 1)
conv_igemm_kernel(const __grid_constant__ TMaps tm, const __grid_constant__ ConvKParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // dynamic smem is only guaranteed 16B-aligned by the API; realign to 1024 for the swizzle atoms.
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);

  const int BN = p.BN;
  const uint32_t a_bytes = kTileM * KC * 2;
  const uint32_t b_bytes = (uint32_t)BN * KC * 2;
  const uint32_t stage_bytes = NP * a_bytes + NP * b_bytes;
  const int S = p.stages;

  // Row-reuse mode (p.yreuse, see the producer): instead of S stages of {A tile, B tile} per (tap, k-chunk) the operand area
  // holds an A ring of p.sa halo tiles (th + kh - 1 image rows: ONE load serves the kh taps of a kernel column) followed by a
  // B ring of p.sb weight tiles.
  const uint32_t a_halo_plane = (uint32_t)p.a_rows * KC * 2;  // one plane of a halo tile
  const uint32_t a_halo_bytes = NP * a_halo_plane;
  const uint32_t b_tile_bytes = NP * b_bytes;
  uint8_t* b_ring = smem + (size_t)p.sa * a_halo_bytes;
  uint8_t* tail = smem + (p.yreuse ? (size_t)p.sa * a_halo_bytes + (size_t)p.sb * b_tile_bytes : (size_t)S * stage_bytes);
  uint64_t* full_bar = (uint64_t*)tail;
  uint64_t* empty_bar = full_bar + kMaxStages;
  uint64_t* afull_bar = empty_bar + kMaxStages;  // row-reuse mode: A ring (full_bar / empty_bar then serve the B ring)
  uint64_t* aempty_bar = afull_bar + kMaxAStages;
  // tile statistics: one slot per (consumer warp, column); every slot has exactly ONE writer per tile, so the CTA's column sums
  // are plain stores summed in a fixed order afterwards (no atomics inside the CTA: reproducible run to run)
  float* col_sum = (float*)(aempty_bar + kMaxAStages);  // [kConsumerWarps][kMaxBN]
  float* col_sq = col_sum + kConsumerWarps * kMaxBN;     // [kConsumerWarps][kMaxBN]
  float* sbias = col_sq + kConsumerWarps * kMaxBN;       // [kMaxBN], p.bias_smem only: zero beyond Cout

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  EMO_STAMP(0, threadIdx.x == 0);

  if (warp == kConsumerWarps) {
    // barrier initialisation and descriptor prefetches spread over the lanes of the producer warp
    if (lane < NP) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tm.a[lane]) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tm.b[lane]) : "memory");
    }
    const int nring = p.yreuse ? p.sb : S;
    if (lane < nring) {
      mbar_init(&full_bar[lane], 1);
      mbar_init(&empty_bar[lane], (uint32_t)kConsumerWarps);  // one arrival per consumer warp
    }
    if (lane >= 16 && lane < 16 + kMaxAStages) {
      mbar_init(&afull_bar[lane - 16], 1);
      mbar_init(&aempty_bar[lane - 16], (uint32_t)kConsumerWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");  // every initialising lane publishes its own barriers
  }
  for (int i = threadIdx.x; i < 2 * kConsumerWarps * kMaxBN; i += kThreads) col_sum[i] = 0.f;
  if (p.bias_smem && threadIdx.x < kMaxBN) {
    const float binv = F16 ? 1.f / p.out_scale : 1.f;  // as the per-tile read below
    sbias[threadIdx.x] = threadIdx.x < BN && (int)threadIdx.x < p.Cout ? __ldg(p.bias + threadIdx.x) * binv : 0.f;
  }
  __syncthreads();
  EMO_STAMP(1, threadIdx.x == 0);
  const int tile_first = (int)blockIdx.x;
  const int tile_step = (int)gridDim.x;
  const int ksplit = p.ksplit;  // work item = tile * ksplit + part (ksplit == 1: item == tile)

  const int taps = p.kd * p.kh * p.kw;
  const int ksteps = taps * p.kchunks;
  const int total_tiles = p.m_tiles * p.n_tiles * p.ksplit;  // work items
  const int rows_a = p.tw * p.th * p.td;
  const uint32_t tx_bytes = (uint32_t)NP * ((uint32_t)rows_a * KC * 2 + b_bytes);

  if (warp >= kConsumerWarps) {
    // the producer warpgroup hands its registers to the consumers; its warps 1..3 have nothing to do
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    if (warp != kConsumerWarps) return;
    // ===================== TMA producer (whole warp walks the loop; one elected lane issues) =====================
    if (p.yreuse) {
      // Row reuse: for a stride-1 convolution the kh taps of one kernel column read the SAME pixels shifted by whole image
      // rows, and in the [row][column][channel] tile a row shift is a whole-swizzle-atom offset (tw x KC x 2 bytes, a multiple
      // of 1024).  So the A operand of a (kernel column, k-chunk) group is loaded ONCE as a halo tile of th + kh - 1 rows and
      // the wgmmas of tap row b read it through a descriptor advanced by b x tw rows: kh times less activation traffic from L2
      // and fewer shared-memory writes per k-step.
      EMO_STAMP(2, lane == 0);
      int sa = 0, sb = 0;
      uint32_t pha = 0, phb = 0;
      const uint32_t a_tx = (uint32_t)NP * a_halo_plane, b_tx = (uint32_t)NP * b_bytes;
      const int ngroups = p.kd * p.kw * p.kchunks;
      for (int item = tile_first; item < total_tiles; item += tile_step) {
        const int nt = item / p.m_tiles;
        int mt = item - nt * p.m_tiles;
        const int twi = mt % p.tiles_w; mt /= p.tiles_w;
        const int thi = mt % p.tiles_h; mt /= p.tiles_h;
        const int tdi = mt % p.tiles_d; mt /= p.tiles_d;
        const int n = mt;
        const int x0 = twi * p.tw - p.pw, y0 = thi * p.th - p.ph, z0 = tdi * p.td - p.pd;
        const int ph = PS ? nt / p.ntc : 0;  // output phase of the sub-pixel form
        const int n0 = (nt - ph * p.ntc) * BN;
        const int xs = (ph & 1) ? 1 : 0, ys = (ph >> 1) ? 1 : 0;
        for (int gi = 0; gi < ngroups; ++gi) {
          const int kc = gi % p.kchunks;
          const int t = gi / p.kchunks;
          const int c = t % p.kw, a = t / p.kw;
          mbar_wait(&aempty_bar[sa], pha ^ 1);
          if (!elect_one()) {
          }
#ifdef EMO_CONV_DEBUG
          else if (p.dbg & 1) {
            mbar_expect_tx(&afull_bar[sa], 0);
          }
#endif
          else {
            uint8_t* dst = smem + (size_t)sa * a_halo_bytes;
            mbar_expect_tx(&afull_bar[sa], a_tx);
#pragma unroll
            for (int pl = 0; pl < NP; ++pl) tma_load_5d(&tm.a[pl], &afull_bar[sa], dst + pl * a_halo_plane, kc * KC, x0 + xs + c, y0 + ys, z0 + a, n);
          }
          __syncwarp();
          if (++sa == p.sa) { sa = 0; pha ^= 1; }
          for (int b = 0; b < p.kh; ++b) {
            const int wtap = PS ? ph * 4 + b * 2 + c : (a * p.kh + b) * p.kw + c;
            mbar_wait(&empty_bar[sb], phb ^ 1);
            if (!elect_one()) {
            }
#ifdef EMO_CONV_DEBUG
            else if (p.dbg & 1) {
              mbar_expect_tx(&full_bar[sb], 0);
            }
#endif
            else {
              uint8_t* dst = b_ring + (size_t)sb * b_tile_bytes;
              mbar_expect_tx(&full_bar[sb], b_tx);
#pragma unroll
              for (int pl = 0; pl < NP; ++pl) tma_load_3d(&tm.b[pl], &full_bar[sb], dst + pl * b_bytes, kc * KC, n0, wtap);
            }
            __syncwarp();
            if (++sb == p.sb) { sb = 0; phb ^= 1; }
          }
        }
      }
      EMO_STAMP(3, lane == 0);
    } else {
      EMO_STAMP(2, lane == 0);
      int stage = 0;
      uint32_t phase = 0;
      for (int item = tile_first; item < total_tiles; item += tile_step) {
        const int tile = item / ksplit, part = item - tile * ksplit;
        const int ks0 = (int)((long long)ksteps * part / ksplit), ks1 = (int)((long long)ksteps * (part + 1) / ksplit);
        const int nt = tile / p.m_tiles;
        int mt = tile - nt * p.m_tiles;
        const int twi = mt % p.tiles_w; mt /= p.tiles_w;
        const int thi = mt % p.tiles_h; mt /= p.tiles_h;
        const int tdi = mt % p.tiles_d; mt /= p.tiles_d;
        const int n = mt;
        const int x0 = twi * p.tw * p.sw - p.pw;
        const int y0 = thi * p.th * p.sh - p.ph;
        const int z0 = tdi * p.td * p.sd - p.pd;
        // sub-pixel form: phase (row parity, column parity) of the output lattice: taps at low-res offsets {-1, 0} for parity 0
        // and {0, +1} for parity 1 (kh = kw = 2 in this mode), weights of this phase at [phase * 4 + tap]
        const int ph = PS ? nt / p.ntc : 0;
        const int n0 = (nt - ph * p.ntc) * BN;
        const int xs = (ph & 1) ? 1 : 0, ys = (ph >> 1) ? 1 : 0;  // p.pw = p.ph = 1: x0 + xs = tile origin - 1 or - 0
        for (int ks = ks0; ks < ks1; ++ks) {
          const int tap = ks / p.kchunks, kc = ks - tap * p.kchunks;
          const int c = tap % p.kw + xs, b = (tap / p.kw) % p.kh + ys, a = PS ? 0 : tap / (p.kw * p.kh);
          const int wtap = ph * 4 + tap;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* st = smem + (size_t)stage * stage_bytes;
          if (!elect_one()) {
          }
#ifdef EMO_CONV_DEBUG
          else if (p.dbg & 1) {
            mbar_expect_tx(&full_bar[stage], 0);
          }
#endif
          else {
            mbar_expect_tx(&full_bar[stage], tx_bytes);
#pragma unroll
            for (int pl = 0; pl < NP; ++pl) {
              tma_load_5d(&tm.a[pl], &full_bar[stage], st + pl * a_bytes, kc * KC, x0 + c, y0 + b, z0 + a, n);
              tma_load_3d(&tm.b[pl], &full_bar[stage], st + NP * a_bytes + pl * b_bytes, kc * KC, n0, wtap);
            }
          }
          __syncwarp();
          if (++stage == S) { stage = 0; phase ^= 1; }
        }
      }
      EMO_STAMP(3, lane == 0);
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
  const int wg = warp >> 2;  // tile rows 64 wg .. 64 wg + 63
  const int wq = warp & 3;   // 16-row slice of the warpgroup's rows
  const int et = threadIdx.x;  // 0..255 among the consumer threads
  const int cq = 2 * (lane & 3);  // first of this thread's two columns in every 8-column block
  const int F = p.flush;
  const uint32_t wg_off = (uint32_t)wg * 64u * KC * 2u;  // the warpgroup's 64 rows inside an A tile
  // The wgmmas of one k-step (KC channels of one tap).  The tensor core accumulates with truncation, so an accumulator only
  // ever takes a short chunk of MMAs (p.flush k-steps, started with scale-d = 0); every chunk is added to the fp32 sums in
  // registers with round-to-nearest adds (DESIGN.md section 2).
  float acc[kMaxBN / 2], cf[kMaxBN / 2];
#pragma unroll
  for (int j = 0; j < kMaxBN / 2; ++j) cf[j] = 0.f;
  auto issue_kstep = [&](auto n_tile, uint32_t sa_, uint32_t a_plane, uint32_t sb_, bool first) {
#ifdef EMO_CONV_DEBUG
    if (p.dbg & 2) return;
#endif
    uint64_t dA[NP], dB[NP];
#pragma unroll
    for (int pl = 0; pl < NP; ++pl) {
      dA[pl] = make_kmajor_desc<KC>(sa_ + pl * a_plane);
      dB[pl] = make_kmajor_desc<KC>(sb_ + pl * b_bytes);
    }
    {
      constexpr int N = decltype(n_tile)::value;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KC / 16; ++kk) {
        const uint64_t adv = (uint64_t)(kk * 2);  // 16 elements = 32 B = 2 x 16B units
        const uint32_t acc0 = (first && kk == 0) ? 0u : 1u;
        if constexpr (NP == 1) {
          wgmma<F16, N>(cf, dA[0] + adv, dB[0] + adv, acc0);
        } else if constexpr (NP == 2) {
          wgmma<F16, N>(cf, dA[1] + adv, dB[0] + adv, acc0);
          wgmma<F16, N>(cf, dA[0] + adv, dB[1] + adv, 1u);
          wgmma<F16, N>(cf, dA[0] + adv, dB[0] + adv, 1u);
        } else {
          // smallest terms first: lo2*hi, hi*lo2, lo*lo, lo*hi, hi*lo, hi*hi
          wgmma<F16, N>(cf, dA[NP - 1] + adv, dB[0] + adv, acc0);
          wgmma<F16, N>(cf, dA[0] + adv, dB[NP - 1] + adv, 1u);
          wgmma<F16, N>(cf, dA[1] + adv, dB[1] + adv, 1u);
          wgmma<F16, N>(cf, dA[1] + adv, dB[0] + adv, 1u);
          wgmma<F16, N>(cf, dA[0] + adv, dB[1] + adv, 1u);
          wgmma<F16, N>(cf, dA[0] + adv, dB[0] + adv, 1u);
        }
      }
      wgmma_commit();
    }
  };
  // One k-step stays in flight while the next is issued: a stage is released once the wgmmas that read it have completed
  // (wait_group 1 after the next k-step's issue); the last k-step of a chunk drains the group before the promotion.
  auto release = [&](uint64_t* bar) {
    __syncwarp();
    if (bar && lane == 0) mbar_arrive(bar);
  };
  auto finish_kstep = [&](bool chunk_last, uint64_t*& pend_b, uint64_t*& pend_a, uint64_t* cur_b, uint64_t* cur_a) {
    if (chunk_last) {
      wgmma_wait<0>();
      wgmma_fence_operands<kMaxBN / 2>(cf);
      release(pend_b); release(pend_a); release(cur_b); release(cur_a);
      pend_b = pend_a = nullptr;
#pragma unroll
      for (int j = 0; j < kMaxBN / 2; ++j) acc[j] += cf[j];
    } else {
      wgmma_wait<1>();
      release(pend_b); release(pend_a);
      pend_b = cur_b; pend_a = cur_a;
    }
  };

  int stage = 0, sa = 0, sb = 0;
  uint32_t phase = 0, pha = 0, phb = 0;
#ifdef EMO_CONV_DEBUG
  long long ph_t = clock64();
#endif
  for (int item = tile_first; item < total_tiles; item += tile_step) {
    const int tile = item / ksplit, part = item - tile * ksplit;
    const int nks = (int)((long long)ksteps * (part + 1) / ksplit) - (int)((long long)ksteps * part / ksplit);
    const int nt = tile / p.m_tiles;
    int mt = tile - nt * p.m_tiles;
    const int twi = mt % p.tiles_w; mt /= p.tiles_w;
    const int thi = mt % p.tiles_h; mt /= p.tiles_h;
    const int tdi = mt % p.tiles_d; mt /= p.tiles_d;
    const int n = mt;
    const int ph = PS ? nt / p.ntc : 0;
    const int n0 = (nt - ph * p.ntc) * BN;
    const int oHt = PS ? p.oH : p.Hout, oWt = PS ? p.oW : p.Wout;  // the output tensor's height and width
    // output coordinates of this thread's row rr (of two) of the tile: valid, flat pixel, residual pixel, spatial index in the sample
    auto locate = [&](int rr, bool& valid, long long& pix, long long& rpix, long long& spi) {
      const int row = wg * 64 + wq * 16 + (lane >> 2) + 8 * rr;  // pixel index inside the tile box
      const int wl = row % p.tw;
      const int hl = (row / p.tw) % p.th;
      const int dl = row / (p.tw * p.th);
      // pixel (gh, gw) of the grid the tiles walk; sub-pixel form: low-res pixel (gh, gw) of phase (pa, pb) -> output pixel
      // (2 gh + pa, 2 gw + pb) of the [oH][oW] output
      const int gw = twi * p.tw + wl, gh = thi * p.th + hl, od = tdi * p.td + dl;
      valid = (row < rows_a) && gw < p.Wout && gh < p.Hout && od < p.Dout;
      const int ow = PS ? 2 * gw + (ph & 1) : gw, oh = PS ? 2 * gh + (ph >> 1) : gh;
      spi = ((long long)od * oHt + oh) * oWt + ow;
      pix = (long long)n * p.Dout * oHt * oWt + spi;
      rpix = p.residual ? (((long long)n * p.rD + od) * p.rH + (oh >> p.res_shift)) * p.rW + (ow >> p.res_shift) : 0;
    };
    // this thread's columns of pixel `pix` of src (residual or post-add) into dst[0 .. BN/4), zero where src or the column
    // does not exist (the even-channel final phase: both columns of a pair exist, 8-byte aligned)
    auto load_pairs = [&](float* dst, const float* src, long long pix, bool valid) {
#pragma unroll
      for (int j = 0; j < kMaxBN / 8; ++j) {
        const int c = n0 + 8 * j + cq;
        float2 v = make_float2(0.f, 0.f);
        if (8 * j < BN && src && valid && c < p.Cout && !EMO_DBG(4)) v = __ldg((const float2*)(src + pix * p.Cout + c));
        dst[2 * j] = v.x; dst[2 * j + 1] = v.y;
      }
    };
    if (ksplit == 1 && (lane & 3) == 0 && (p.residual || p.post_add)) {
      // the residual / post-add rows are first read after this tile's main loop: pull them into L2 now
      const int nb = (BN < p.Cout - n0 ? BN : p.Cout - n0) * 4;
      for (int rr = 0; rr < 2; ++rr) {
        bool valid;
        long long pix, rpix, spi;
        locate(rr, valid, pix, rpix, spi);
        if (!valid) continue;
        if (p.residual) {
          const char* rp = (const char*)(p.residual + rpix * p.Cout + n0);
          for (int b = 0; b < nb; b += 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(rp + b));
        }
        if (p.post_add) {
          const char* rp = (const char*)(p.post_add + spi * p.Cout + n0);
          for (int b = 0; b < nb; b += 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(rp + b));
        }
      }
    }

    // ---- fp32 register accumulation of the short wgmma chunks, starting from the bias (un-split layers) ----
    if (p.bias && ksplit == 1) {
      // fp16 operands: the sums are multiplied by out_scale (a power of two) below: exact
      const float binv = F16 ? 1.f / p.out_scale : 1.f;
#pragma unroll
      for (int j = 0; j < kMaxBN / 8; ++j) {
        const int c = n0 + 8 * j + cq;
        float b0 = 0.f, b1 = 0.f;
        if (8 * j < BN) {
          if (p.bias_smem) {
            const float2 b = *(const float2*)(sbias + c);  // n0 == 0
            b0 = b.x; b1 = b.y;
          } else {
            if (c < p.Cout) b0 = __ldg(p.bias + c) * binv;
            if (c + 1 < p.Cout) b1 = __ldg(p.bias + c + 1) * binv;
          }
        }
        acc[4 * j] = b0; acc[4 * j + 1] = b1; acc[4 * j + 2] = b0; acc[4 * j + 3] = b1;
      }
    } else {
#pragma unroll
      for (int j = 0; j < kMaxBN / 2; ++j) acc[j] = 0.f;
    }
    EMO_PHASE(5);

    uint64_t* pend_b = nullptr;
    uint64_t* pend_a = nullptr;
    // the main loop is instantiated per N tile width: the k-steps are then straight-line wgmma code of one shape
    wgmma_dispatch_n(BN, [&](auto n_tile) {
    if (p.yreuse) {
      const int ngroups = p.kd * p.kw * p.kchunks;
      const uint32_t row_shift = (uint32_t)p.tw * KC * 2;  // one image row of the halo tile: a whole number of swizzle atoms
      int ks = 0;
      for (int gi = 0; gi < ngroups; ++gi) {
        EMO_PHASE(1);
        mbar_wait(&afull_bar[sa], pha);
        EMO_PHASE(0);
        EMO_STAMP(4, et == 0 && item == tile_first && gi == 0);
        for (int b = 0; b < p.kh; ++b, ++ks) {
          const bool chunk_first = (ks % F) == 0;
          const bool chunk_last = ((ks + 1) % F) == 0 || ks == nks - 1;
          EMO_PHASE(1);
          mbar_wait(&full_bar[sb], phb);
          EMO_PHASE(0);
          issue_kstep(n_tile, smem_u32(smem + (size_t)sa * a_halo_bytes) + (uint32_t)b * row_shift + wg_off, a_halo_plane,
                      smem_u32(b_ring + (size_t)sb * b_tile_bytes), chunk_first);
          // the halo tile is released with the last of its kh tap rows
          finish_kstep(chunk_last, pend_b, pend_a, &empty_bar[sb], b == p.kh - 1 ? &aempty_bar[sa] : nullptr);
          if (++sb == p.sb) { sb = 0; phb ^= 1; }
        }
        if (++sa == p.sa) { sa = 0; pha ^= 1; }
      }
    } else {
      for (int ks = 0; ks < nks; ++ks) {
        const bool chunk_first = (ks % F) == 0;
        const bool chunk_last = ((ks + 1) % F) == 0 || ks == nks - 1;
        EMO_PHASE(1);
        mbar_wait(&full_bar[stage], phase);
        EMO_PHASE(0);
        EMO_STAMP(4, et == 0 && item == tile_first && ks == 0);
        const uint32_t st = smem_u32(smem + (size_t)stage * stage_bytes);
        issue_kstep(n_tile, st + wg_off, a_bytes, st + NP * a_bytes, chunk_first);
        finish_kstep(chunk_last, pend_b, pend_a, &empty_bar[stage], nullptr);
        if (++stage == S) { stage = 0; phase ^= 1; }
      }
    }
    });
    EMO_STAMP(5, et == 0);
    if constexpr (F16) {
      // the operand planes carried power-of-two scales (activations x sa, weights x sw): undo them on the fp32 sums (exact)
#pragma unroll
      for (int j = 0; j < kMaxBN / 2; ++j) acc[j] *= p.out_scale;
    }
    EMO_PHASE(1);
#ifdef EMO_CONV_DEBUG
    if ((p.dbg & 512) && et == 0 && blockIdx.x < 160) atomicAdd(&g_conv_phase[blockIdx.x * 8 + 7], 1ull);
#endif

    // ---- final phase: this thread's two rows ----
    if (ksplit > 1) {
      // split-K: this part's partial tile goes to ITS OWN slice of the fp32 workspace (plain stores: every output element
      // is written exactly once per part); the finalize kernel sums the parts in part order - a fixed order, so the result
      // does not depend on which CTA finished first - and applies bias / residual / activation / statistics
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        bool valid;
        long long pix, rpix, spi;
        locate(rr, valid, pix, rpix, spi);
        if (!valid) continue;
        float* wrow = p.ws + (size_t)part * (size_t)p.ws_part_elems + pix * p.Cout;
#pragma unroll
        for (int j = 0; j < kMaxBN / 8; ++j) {
          const int c = n0 + 8 * j + cq;
          if (8 * j < BN) {
            if (c < p.Cout) wrow[c] = acc[4 * j + 2 * rr];
            if (c + 1 < p.Cout) wrow[c + 1] = acc[4 * j + 2 * rr + 1];
          }
        }
      }
      EMO_PHASE(3);
      continue;
    }
    const long long sp = (long long)p.Dout * oHt * oWt;
    // The final phase is unrolled over the 8-column blocks and both rows, so its code is long.  It is instantiated once per
    // activation, with the odd-channel scalar path in an instantiation of its own: a tile then runs straight-line code that
    // holds only what it executes.  A run-time activation switch and the scalar path inside every block would scatter the
    // executed instructions over far more code than the instruction caches hold, fetched anew by every tile (DESIGN.md
    // section 7).
    auto final_rows = [&](auto pairs_c, auto act_c) {
      constexpr bool pairs = decltype(pairs_c)::value;  // c even, Cout even: both columns of a pair exist, 8-byte aligned
      constexpr int act_k = decltype(act_c)::value;
      const int act = act_k >= 0 ? act_k : p.act;  // -1: the activation is read at run time (the scalar path)
      if constexpr (pairs) {
        // The residual / post-add values are loaded before the stores they precede: a load may not move over a store that may
        // alias it, so a load after a store waits out a full memory latency.  They go to the chunk registers, which are free
        // until the next tile's main loop: both rows' residual at once when there is no post-add (every residual layer of the
        // models), otherwise one row's residual and post-add at a time.
        bool valid[2];
        long long pix[2], rpix[2], spi[2];
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) locate(rr, valid[rr], pix[rr], rpix[rr], spi[rr]);
        auto loads_landed = [&] {
#ifdef EMO_CONV_DEBUG
          if (p.dbg & 512) {
            // phase clocks: wait for the loads here, so that their latency is counted as load time
            float s = 0.f;
#pragma unroll
            for (int j = 0; j < kMaxBN / 2; ++j) s += cf[j];
            if (s == 1.2345e-38f) g_conv_phase[0] = 0;
          }
#endif
          EMO_PHASE(2);
        };
        // act(v + residual), then the post-add as a separate rounding (__fadd_rn: never contracted into the activation's
        // last multiply; + 0 without one), then the stores; zero outside the tensor, so that those pixels / channels are no
        // part of the statistics
        auto finish_row = [&](int rr, const float* res, const float* post) {
#pragma unroll
          for (int j = 0; j < kMaxBN / 8; ++j) {
            if (8 * j >= BN) continue;
            const int c = n0 + 8 * j + cq;
            float v0 = 0.f, v1 = 0.f;
            if (valid[rr] && c < p.Cout && !EMO_DBG(8)) {
              v0 = __fadd_rn(act_apply(acc[4 * j + 2 * rr] + res[2 * j], act), post ? post[2 * j] : 0.f);
              v1 = __fadd_rn(act_apply(acc[4 * j + 2 * rr + 1] + res[2 * j + 1], act), post ? post[2 * j + 1] : 0.f);
              if (!p.out_nchw) {
                *(float2*)(p.out + pix[rr] * p.Cout + c) = make_float2(v0, v1);
              } else {
                p.out[((long long)n * p.Cout + c) * sp + spi[rr]] = v0;
                p.out[((long long)n * p.Cout + c + 1) * sp + spi[rr]] = v1;
              }
            }
            acc[4 * j + 2 * rr] = v0; acc[4 * j + 2 * rr + 1] = v1;
          }
        };
        if (!p.post_add) {
          load_pairs(cf, p.residual, rpix[0], valid[0]);
          load_pairs(cf + kMaxBN / 4, p.residual, rpix[1], valid[1]);
          loads_landed();
          finish_row(0, cf, nullptr);
          finish_row(1, cf + kMaxBN / 4, nullptr);
        } else {
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            load_pairs(cf, p.residual, rpix[rr], valid[rr]);
            load_pairs(cf + kMaxBN / 4, p.post_add, spi[rr], valid[rr]);
            loads_landed();
            finish_row(rr, cf, cf + kMaxBN / 4);
            EMO_PHASE(3);
          }
        }
        if (!p.post_add) EMO_PHASE(3);
      } else {
        // odd channel count (e.g. Cout = 3): scalar path
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          bool valid;
          long long pix, rpix, spi;
          locate(rr, valid, pix, rpix, spi);
          EMO_PHASE(2);
#pragma unroll
          for (int j = 0; j < kMaxBN / 8; ++j) {
            if (8 * j >= BN) continue;
            const int c = n0 + 8 * j + cq;
#pragma unroll
            for (int q = 0; q < 2; ++q) {
              const int cc = c + q;
              float x = acc[4 * j + 2 * rr + q];
              if (valid && cc < p.Cout && !EMO_DBG(8)) {
                if (p.residual) x += __ldg(p.residual + rpix * p.Cout + cc);
                x = act_apply(x, act);
                if (p.post_add) x += __ldg(p.post_add + spi * p.Cout + cc);
                if (!p.out_nchw) p.out[pix * p.Cout + cc] = x;
                else p.out[((long long)n * p.Cout + cc) * sp + spi] = x;
              } else {
                x = 0.f;  // pixels / channels outside the tensor: no part of the statistics
              }
              acc[4 * j + 2 * rr + q] = x;
            }
          }
          EMO_PHASE(3);
        }
      }
    };
    using std::integral_constant;
    if ((p.Cout & 1) != 0) {
      final_rows(std::false_type{}, integral_constant<int, -1>{});
    } else {
      switch (p.act) {
        case EMO_ACT_RELU: final_rows(std::true_type{}, integral_constant<int, EMO_ACT_RELU>{}); break;
        case EMO_ACT_SIGMOID: final_rows(std::true_type{}, integral_constant<int, EMO_ACT_SIGMOID>{}); break;
        case EMO_ACT_TANH: final_rows(std::true_type{}, integral_constant<int, EMO_ACT_TANH>{}); break;
        default: final_rows(std::true_type{}, integral_constant<int, EMO_ACT_NONE>{}); break;
      }
    }
    EMO_STAMP(6, et == 0);

    if (p.stats && !EMO_DBG(16)) {
      // column sums of the warp's 16 rows: two rows in the thread, then a butterfly over the eight lanes sharing the columns
      float* cs = col_sum + warp * kMaxBN;
      float* cqs = col_sq + warp * kMaxBN;
#pragma unroll
      for (int j = 0; j < kMaxBN / 8; ++j) {
        if (8 * j >= BN) continue;
        float s0 = acc[4 * j] + acc[4 * j + 2], s1 = acc[4 * j + 1] + acc[4 * j + 3];
        float q0 = acc[4 * j] * acc[4 * j] + acc[4 * j + 2] * acc[4 * j + 2];
        float q1 = acc[4 * j + 1] * acc[4 * j + 1] + acc[4 * j + 3] * acc[4 * j + 3];
#pragma unroll
        for (int off = 4; off < 32; off <<= 1) {
          s0 += __shfl_xor_sync(0xffffffffu, s0, off);
          s1 += __shfl_xor_sync(0xffffffffu, s1, off);
          q0 += __shfl_xor_sync(0xffffffffu, q0, off);
          q1 += __shfl_xor_sync(0xffffffffu, q1, off);
        }
        if (lane < 4) {
          cs[8 * j + cq] = s0; cs[8 * j + cq + 1] = s1;
          cqs[8 * j + cq] = q0; cqs[8 * j + cq + 1] = q1;
        }
      }
      asm volatile("bar.sync 1, %0;" ::"n"(kConsumerWarps * 32) : "memory");
      tile_group_stats(p, col_sum, col_sq, n, n0, BN, et, kConsumerWarps * 32);
      asm volatile("bar.sync 1, %0;" ::"n"(kConsumerWarps * 32) : "memory");  // the slots are rewritten by the next tile
    }
    EMO_PHASE(4);
    EMO_STAMP(7, et == 0);
  }
  EMO_STAMP(8, et == 0);
}

// split-K finalize: out = act(sum_parts ws[part] + bias + residual) + post_add, statistics.  The parts are summed in part
// order (fixed), so the output is reproducible run to run.
struct FinParams {
  const float* ws;
  int ksplit;
  long long part_elems;
  float* out;
  int N, C;
  long long S;  // spatial positions per sample
  const float* bias;
  const float* residual;
  const float* post_add;
  int act, out_nchw;
  double* stats;
  int G;
};

__global__ void __launch_bounds__(256) splitk_finalize_kernel(const FinParams f) {
  extern __shared__ double sstat[];  // fp64: sums of fp32 values are exact -> independent of the order of the atomics
  const int n = blockIdx.y;
  if (f.stats) {
    for (int i = threadIdx.x; i < 2 * f.G; i += blockDim.x) sstat[i] = 0.0;
    __syncthreads();
  }
  const long long per_n = f.S * f.C;
  const int cpg = f.stats ? f.C / f.G : 1;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < per_n; t += (long long)gridDim.x * blockDim.x) {
    const long long i = (long long)n * per_n + t;
    const int c = (int)(t % f.C);
    const long long sp = t / f.C;
    float v = 0.f;
#pragma unroll 8
    for (int k = 0; k < f.ksplit; ++k) v += __ldcg(f.ws + (long long)k * f.part_elems + i);  // part order: reproducible
    if (f.bias) v += __ldg(f.bias + c);
    if (f.residual) v += __ldg(f.residual + i);
    v = act_apply(v, f.act);
    if (f.post_add) v += __ldg(f.post_add + t);
    if (f.out_nchw) f.out[((long long)n * f.C + c) * f.S + sp] = v;
    else f.out[i] = v;
    if (f.stats) {
      atomicAdd(&sstat[c / cpg], (double)v);
      atomicAdd(&sstat[f.G + c / cpg], (double)(v * v));
    }
  }
  if (f.stats) {
    __syncthreads();
    for (int g = threadIdx.x; g < f.G; g += blockDim.x) {
      atomicAdd(&f.stats[((long long)n * f.G + g) * 2], sstat[g]);
      atomicAdd(&f.stats[((long long)n * f.G + g) * 2 + 1], sstat[f.G + g]);
    }
  }
}

// Fused finalize + normalisation + activation + plane split for SMALL split-K layers (emo_conv_desc.post): one 8-CTA
// cluster per sample does what splitk_finalize_kernel + gn statistics + emo_apply do in three launches for the ResNet
// tails and the first warp-generator blocks (<= 64 Ki elements per sample, 4x4 .. 32x32 maps), whose time is launch
// latency, not work.  Thread -> elements e = rank * 512 + tid + k * 4096: C divides 512, so a thread owns ONE channel.
// GroupNorm statistics: per-thread sums in element order -> per-CTA group sums in thread order -> cluster totals in rank
// order over distributed shared memory: fixed orders throughout, bit-reproducible.
static constexpr int kPostCluster = 8;
static constexpr int kPostThreads = 512;
static constexpr int kPostMaxV = 16;  // elements per thread: <= 65536 elements per sample
struct PostParams {
  const float* ws;
  int ksplit;
  long long part_elems;
  int N, C;
  long long S;
  const float* bias;      // the convolution's own bias / same-resolution residual / activation (before the norm)
  const float* residual;
  int conv_act;
  emo_apply_desc ap;      // the post-op: x ignored (= the convolution's output), up == 1
};

__device__ __forceinline__ uint32_t dsmem_addr(const void* local, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(local)), "r"(rank));
  return r;
}
__device__ __forceinline__ double ld_dsmem_f64(uint32_t addr) {
  double v;
  asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(addr) : "memory");
  return v;
}

__global__ void __launch_bounds__(kPostThreads, 1) splitk_post_kernel(const PostParams f) {
  __shared__ float s_sum[kPostThreads], s_sq[kPostThreads];
  __shared__ double s_part[2 * 64];  // this CTA's (sum, sum of squares) per group
  __shared__ double s_tot[2 * 64];   // cluster totals
  const emo_apply_desc& a = f.ap;
  const int tid = threadIdx.x;
  const uint32_t rank = (uint32_t)blockIdx.x % kPostCluster;
  const int n = (int)blockIdx.x / kPostCluster;
  const long long per_n = f.S * f.C;
  const int c = tid % f.C;  // this thread's channel (512 % C == 0 and 4096 % C == 0)
  float v[kPostMaxV];
  float ts = 0.f, tq = 0.f;
  const long long e0 = (long long)rank * kPostThreads + tid;               // this thread's elements: e0 + k * 4096
  const long long base = (long long)n * per_n;
#pragma unroll
  for (int k = 0; k < kPostMaxV; ++k) v[k] = 0.f;
  // K parts summed in part order; four parts x all of the thread's elements are loaded before they are added, so up to 64
  // independent L2 loads are in flight per thread instead of one (ncu, round 2: 26 us per launch with the serial loop)
  for (int part = 0; part < f.ksplit; part += 4) {
    float t[4][kPostMaxV];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float* w = f.ws + (long long)(part + q) * f.part_elems + base;
#pragma unroll
      for (int k = 0; k < kPostMaxV; ++k) {
        const long long e = e0 + (long long)k * (kPostCluster * kPostThreads);
        t[q][k] = (part + q < f.ksplit && e < per_n) ? __ldcg(w + e) : 0.f;
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int k = 0; k < kPostMaxV; ++k) v[k] += t[q][k];
  }
#pragma unroll
  for (int k = 0; k < kPostMaxV; ++k) {
    const long long e = e0 + (long long)k * (kPostCluster * kPostThreads);
    if (e < per_n) {
      const long long i = base + e;
      float x = v[k];
      if (f.bias) x += __ldg(f.bias + c);
      if (f.residual) x += __ldg(f.residual + i);
      x = act_apply(x, f.conv_act);
      v[k] = x;
      ts += x; tq = fmaf(x, x, tq);
    } else {
      v[k] = 0.f;
    }
  }
  float A = 1.f, B = 0.f;
  if (a.stats) {
    // GroupNorm of the convolution's output
    const int G = a.G, cpg = f.C / G;
    s_sum[tid] = ts; s_sq[tid] = tq;
    __syncthreads();
    if (tid < G) {
      double sg = 0.0, qg = 0.0;
      for (int m = 0; m < kPostThreads / f.C; ++m)
        for (int cc = tid * cpg; cc < (tid + 1) * cpg; ++cc) { sg += (double)s_sum[cc + m * f.C]; qg += (double)s_sq[cc + m * f.C]; }
      s_part[tid] = sg; s_part[64 + tid] = qg;
    }
    cluster_sync_all();  // every CTA's group sums are in its shared memory
    if (tid < G) {
      double sg = 0.0, qg = 0.0;
      for (uint32_t r = 0; r < (uint32_t)kPostCluster; ++r) {
        sg += ld_dsmem_f64(dsmem_addr(&s_part[tid], r));
        qg += ld_dsmem_f64(dsmem_addr(&s_part[64 + tid], r));
      }
      s_tot[tid] = sg; s_tot[64 + tid] = qg;
      if (rank == 0) {  // publish the statistics too (same layout as every other producer)
        double* st = const_cast<double*>(a.stats);  // == the convolution's `stats` output (checked by the host)
        st[((long long)n * G + tid) * 2] = sg;
        st[((long long)n * G + tid) * 2 + 1] = qg;
      }
    }
    cluster_sync_all();  // nobody retires (or overwrites s_part) while a peer may still read it
    const int g = c / cpg;
    const double mean = s_tot[g] / a.count;
    double var = s_tot[64 + g] / a.count - mean * mean;
    if (var < 0) var = 0;
    const float rstd = (float)(1.0 / sqrt(var + (double)a.eps));
    float gam = a.gamma ? a.gamma[c] : 1.f, bet = a.beta ? a.beta[c] : 0.f;
    if (a.ada_w) {
      const float aw = a.ada_w[(long long)n * f.C + c], ab = a.ada_b[(long long)n * f.C + c];
      bet = bet * aw + ab;
      gam = gam * aw;
    }
    A = rstd * gam;
    B = bet - (float)mean * A;
  } else if (a.A) {
    A = a.A[(a.ab_per_sample ? (long long)n * f.C : 0) + c];
    B = a.B[(a.ab_per_sample ? (long long)n * f.C : 0) + c];
  }
  float A2 = 1.f, B2 = 0.f;
  if (a.A2) { A2 = a.A2[c]; B2 = a.B2[c]; }
#pragma unroll
  for (int k = 0; k < kPostMaxV; ++k) {
    const long long e = (long long)rank * kPostThreads + tid + (long long)k * (kPostCluster * kPostThreads);
    if (e < per_n) {
      const long long i = (long long)n * per_n + e;
      float y = fmaf(v[k], A, B);
      if (a.res) y += fmaf(__ldg(a.res + i), A2, B2);
      y = act_apply(y, a.act);
      if (a.out) a.out[i] = y;
      if (a.out_hi) {
        if (a.plane_fp16 && !a.out_lo) {
          ((__half*)a.out_hi)[i] = f16_plane(y * a.plane_scale);
        } else if (a.plane_fp16) {
          __half h, l;
          split_f16(y * a.plane_scale, h, l);
          ((__half*)a.out_hi)[i] = h; ((__half*)a.out_lo)[i] = l;
        } else if (a.out_lo2) {
          __nv_bfloat16 h, l, l2;
          split_bf16x3(y, h, l, l2);
          ((__nv_bfloat16*)a.out_hi)[i] = h; ((__nv_bfloat16*)a.out_lo)[i] = l; ((__nv_bfloat16*)a.out_lo2)[i] = l2;
        } else {
          __nv_bfloat16 h, l;
          split_bf16(y, h, l);
          ((__nv_bfloat16*)a.out_hi)[i] = h; ((__nv_bfloat16*)a.out_lo)[i] = l;
        }
      }
    }
  }
}


// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static PFN_cuTensorMapEncodeTiled get_encode() {
  static PFN_cuTensorMapEncodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || !p) return nullptr;
    fn = (PFN_cuTensorMapEncodeTiled)p;
  }
  return fn;
}

static int pick_box(int dim, int want) {
  int b = want;
  while (b > dim) b >>= 1;
  return b < 1 ? 1 : b;
}

// The kernel instantiations, indexed by EMO_CONV_KERNEL_*: plan_conv picks a row, emo_conv_igemm launches that row's kernel.
struct ConvKernel {
  int KC, NP;
  bool ps, f16;
  void (*fn)(TMaps, ConvKParams);
};
static const ConvKernel kConvKernels[] = {
    {64, 2, false, false, conv_igemm_kernel<64, 2, false, false>},  // EMO_CONV_KERNEL_BF16X2_KC64
    {32, 2, false, false, conv_igemm_kernel<32, 2, false, false>},  // EMO_CONV_KERNEL_BF16X2_KC32
    {64, 3, false, false, conv_igemm_kernel<64, 3, false, false>},  // EMO_CONV_KERNEL_BF16X3_KC64
    {32, 3, false, false, conv_igemm_kernel<32, 3, false, false>},  // EMO_CONV_KERNEL_BF16X3_KC32
    {64, 2, false, true, conv_igemm_kernel<64, 2, false, true>},    // EMO_CONV_KERNEL_F16_KC64
    {32, 2, false, true, conv_igemm_kernel<32, 2, false, true>},    // EMO_CONV_KERNEL_F16_KC32
    {64, 2, true, false, conv_igemm_kernel<64, 2, true, false>},    // EMO_CONV_KERNEL_UPCONV_KC64
    {64, 1, false, true, conv_igemm_kernel<64, 1, false, true>},    // EMO_CONV_KERNEL_H1_KC64
    {32, 1, false, true, conv_igemm_kernel<32, 1, false, true>},    // EMO_CONV_KERNEL_H1_KC32
    {64, 1, true, true, conv_igemm_kernel<64, 1, true, true>},      // EMO_CONV_KERNEL_H1_UPCONV_KC64
};
static constexpr int kNumConvKernels = (int)(sizeof(kConvKernels) / sizeof(kConvKernels[0]));
static_assert(kNumConvKernels == EMO_CONV_KERNEL_H1_UPCONV_KC64 + 1, "one row per EMO_CONV_KERNEL_* id");

// What emo_conv_igemm runs for one descriptor: the kernel parameters (tiles, N tile, k-chunk, pipeline depths, split-K,
// accumulation chunk), the kernel form, the grid, the shared-memory size and the launches that finish the convolution.
struct ConvPlan {
  ConvKParams p;
  int NP, KC, f16, ps, kh_eff;
  int kernel;  // EMO_CONV_KERNEL_*
  int grid;
  int finish;  // EMO_CONV_FINISH_*
  size_t smem_bytes;
};

// Checks the descriptor and plans the launch for a device of `sm_count` SMs.  Host arithmetic only (no CUDA call): emo_conv_plan
// reports the same plan without a device.
static int plan_conv(const emo_conv_desc* d, int sm_count, ConvPlan* plan) {
  EMO_REQUIRE(plan && sm_count >= 1, "emo_conv_igemm: bad plan arguments (sm_count=%d)", sm_count);
  memset(plan, 0, sizeof(*plan));
  ConvKParams& p = plan->p;
  // one-plane fp16 operands: a_lo == w_lo == NULL with operand_fp16 (a_lo2 / w_lo2 then must be NULL too)
  const bool one_plane = d && !d->a_lo && !d->w_lo;
  EMO_REQUIRE(d && d->a_hi && d->w_hi && d->out && (one_plane || (d->a_lo && d->w_lo)),
              "emo_conv_igemm: null pointer (a_lo and w_lo are both given, or both NULL for one-plane fp16 operands)");
  EMO_REQUIRE(!one_plane || (d->operand_fp16 && !d->a_lo2 && !d->w_lo2),
              "emo_conv_igemm: one-plane operands (a_lo == w_lo == NULL) are fp16 only (operand_fp16) and take no a_lo2 / w_lo2");
  EMO_REQUIRE(d->Cin % 32 == 0, "emo_conv_igemm: Cin=%d must be a multiple of 32 (use emo_conv_direct)", d->Cin);
  EMO_REQUIRE(d->Cout_pad % 16 == 0 && d->Cout <= d->Cout_pad, "emo_conv_igemm: Cout_pad=%d must be a multiple of 16 >= Cout", d->Cout_pad);
  EMO_REQUIRE(d->sd >= 1 && d->sh >= 1 && d->sw >= 1 && d->sd <= 2 && d->sh <= 2 && d->sw <= 2, "emo_conv_igemm: stride must be 1 or 2");
  EMO_REQUIRE(((uintptr_t)d->a_hi % 16) == 0 && ((uintptr_t)d->a_lo % 16) == 0 && ((uintptr_t)d->w_hi % 16) == 0 &&
                  ((uintptr_t)d->w_lo % 16) == 0 && ((uintptr_t)d->out % 16) == 0,
              "emo_conv_igemm: pointers must be 16-byte aligned");
  if (d->stats) EMO_REQUIRE(d->G > 0 && d->Cout % d->G == 0, "emo_conv_igemm: Cout=%d not divisible by G=%d", d->Cout, d->G);
  if (d->post) {
    EMO_REQUIRE(!d->out_nchw && d->post->N == d->N && d->post->C == d->Cout && d->post->D == d->Dout && d->post->H == d->Hout && d->post->W == d->Wout,
                "emo_conv_igemm: post-op shape must be the convolution's channels-last output shape");
    EMO_REQUIRE(!d->post->stats || d->post->stats == d->stats, "emo_conv_igemm: a GroupNorm post-op normalises with the convolution's own statistics (post->stats == stats)");
  }
  const bool vec_ok = (d->Cout % 4 == 0);
  EMO_REQUIRE(vec_ok || d->Cout < 16, "emo_conv_igemm: Cout=%d must be a multiple of 4 (or < 16)", d->Cout);

  const int NP = one_plane ? 1 : d->a_lo2 ? 3 : 2;
  EMO_REQUIRE((d->a_lo2 == nullptr) == (d->w_lo2 == nullptr), "emo_conv_igemm: a_lo2 and w_lo2 must be given together");
  // sub-pixel mode: the descriptor describes conv3x3(pad 1)(nearest_x2(input)) with the input given at LOW resolution and
  // the weights pre-folded to [4 phases][2x2 taps][Cout_pad][Cin] (emoportraits_b200/ops.py: pack_upconv_weight)
  const int ps = d->upconv ? 1 : 0;
  if (ps) {
    EMO_REQUIRE(d->kd == 1 && d->kh == 3 && d->kw == 3 && d->sd == 1 && d->sh == 1 && d->sw == 1 && d->pd == 0 && d->ph == 1 && d->pw == 1,
                "emo_conv_igemm: upconv needs a 1x3x3 stride-1 pad-1 convolution");
    EMO_REQUIRE(d->Din == 1 && d->Dout == 1 && d->Hout == 2 * d->Hin && d->Wout == 2 * d->Win,
                "emo_conv_igemm: upconv output must be (2 Hin, 2 Win) (got %d x %d from %d x %d)", d->Hout, d->Wout, d->Hin, d->Win);
    EMO_REQUIRE(NP <= 2 && d->Cin % 64 == 0 && d->Cout == d->Cout_pad && !d->out_nchw,
                "emo_conv_igemm: upconv needs two-plane bf16 or one-plane fp16 operands, Cin %% 64 == 0, Cout %% 16 == 0, channels-last output");
  }
  const int f16 = d->operand_fp16 ? 1 : 0;
  if (f16) EMO_REQUIRE(NP <= 2 && !(ps && NP == 2) && d->out_scale > 0.f,
                       "emo_conv_igemm: fp16 operands need one or two planes (upconv: one), out_scale > 0");
  const int gH = ps ? d->Hin : d->Hout, gW = ps ? d->Win : d->Wout;  // the pixel grid the tiles walk
  const int taps_k = ps ? 4 : d->kd * d->kh * d->kw;                  // taps in one tile's K loop
  const int nt_mult = ps ? 4 : 1;                                     // N tiles per channel tile (one per output phase)
  int KC = (d->Cin % 64 == 0) ? 64 : 32;  // three-plane tiles fall back to 32 below when 64 leaves < 3 pipeline stages
  // N tile: largest multiple of 16 that divides Cout_pad and fits the register-resident accumulators
  int BN = 0;
  for (int cand = kMaxBN; cand >= 16; cand -= 16)
    if (d->Cout_pad % cand == 0) { BN = cand; break; }
  EMO_REQUIRE(BN > 0, "emo_conv_igemm: no N tile for Cout_pad=%d", d->Cout_pad);

  p.N = d->N; p.Dout = d->Dout; p.Hout = gH; p.Wout = gW; p.Cout = d->Cout;
  p.oH = d->Hout; p.oW = d->Wout;
  p.kd = d->kd; p.kh = ps ? 2 : d->kh; p.kw = ps ? 2 : d->kw; p.sd = d->sd; p.sh = d->sh; p.sw = d->sw;
  p.pd = d->pd; p.ph = d->ph; p.pw = d->pw;
  // pixel box: 128 pixels, widest along W first
  p.tw = pick_box(gW, 16);
  p.th = pick_box(gH, kTileM / p.tw > 0 ? kTileM / p.tw : 1);
  p.td = pick_box(d->Dout, kTileM / (p.tw * p.th) > 0 ? kTileM / (p.tw * p.th) : 1);
  if (p.tw * p.th * p.td < kTileM && p.tw < gW) {  // shallow/short tensor: widen along W
    int tw = p.tw;
    while (tw * 2 <= gW && tw * 2 * p.th * p.td <= kTileM && tw * 2 * d->sw <= 256) tw *= 2;
    p.tw = tw;
  }
  EMO_REQUIRE(p.tw * d->sw <= 256 && p.th * d->sh <= 256 && p.td * d->sd <= 256, "emo_conv_igemm: TMA box too large");
  p.tiles_w = cdiv(gW, p.tw); p.tiles_h = cdiv(gH, p.th); p.tiles_d = cdiv(d->Dout, p.td);
  p.m_tiles = d->N * p.tiles_d * p.tiles_h * p.tiles_w;
  // small-M layers (ResNet tails, the first warp-generator blocks): the serial K loop of a handful of CTAs is bound by the
  // TMA -> MMA round trip, not by work.  With a workspace: split K over CTAs (one fp32 workspace slice per part, finalize
  // pass).  Without: narrow the N tile until the tile count fills the machine.
  const int ksteps_total = taps_k * (d->Cin / ((d->Cin % 64 == 0) ? 64 : 32));
  int ksplit = 1;
  {
    const long long tiles = (long long)p.m_tiles * (d->Cout_pad / BN) * nt_mult;
    const long long out_elems = (long long)d->N * d->Dout * d->Hout * d->Wout * d->Cout;
    if (!ps && d->splitk_ws && 2 * out_elems <= d->splitk_ws_elems && d->res_shift == 0 && tiles * 2 <= sm_count) {
      long long parts = (2ll * sm_count) / tiles;
      if (parts > ksteps_total / 4) parts = ksteps_total / 4;
      if (parts * out_elems > d->splitk_ws_elems) parts = d->splitk_ws_elems / out_elems;  // one workspace slice per part
      if (parts >= 2) ksplit = (int)parts;
    }
  }
  if (ksplit == 1 && (long long)p.m_tiles * (d->Cout_pad / BN) * nt_mult < sm_count / 2) {
    for (int cand = BN; cand >= 16; cand -= 16) {
      if (d->Cout_pad % cand) continue;
      BN = cand;
      if ((long long)p.m_tiles * (d->Cout_pad / cand) * nt_mult >= sm_count) break;
    }
  }
  p.BN = BN;
  p.ntc = d->Cout_pad / BN;
  p.n_tiles = p.ntc * nt_mult;
  p.ksplit = ksplit;
  p.ws = d->splitk_ws;
  p.ws_part_elems = (long long)d->N * d->Dout * d->Hout * d->Wout * d->Cout;
  p.dbg = 0;
#ifdef EMO_CONV_DEBUG
  { const char* e = getenv("EMO_CONV_DBG"); p.dbg = e ? atoi(e) : 0; }
#endif
  p.bias = d->bias; p.residual = d->residual; p.res_shift = d->res_shift; p.act = d->act;
  p.rD = d->Dout; p.rH = d->Hout >> d->res_shift; p.rW = d->Wout >> d->res_shift;
  p.post_add = d->post_add; p.out = d->out; p.out_nchw = d->out_nchw;
  p.stats = d->stats; p.G = d->G; p.cpg = d->G > 0 ? d->Cout / d->G : 1;
  p.out_scale = f16 ? d->out_scale : 1.f;
  EMO_REQUIRE(!d->residual || ((d->Hout % (1 << d->res_shift)) == 0 && (d->Wout % (1 << d->res_shift)) == 0),
              "emo_conv_igemm: residual shift does not divide the output size");

  const size_t tail_bytes = (2 * kMaxStages + 2 * kMaxAStages) * 8 + 2 * kConsumerWarps * kMaxBN * sizeof(float);
  const size_t smem_limit = 227 * 1024;  // the sm_90 opt-in maximum per block
  const size_t avail = smem_limit - tail_bytes - 1024;
  const int KC0 = KC;
  if (KC == 64 && avail / ((size_t)NP * (kTileM + BN) * 64 * 2) < 3) KC = 32;
  const size_t stage_bytes = (size_t)NP * (kTileM + BN) * KC * 2;
  int stages = (int)(avail / stage_bytes);
  // row reuse needs: more than one tap row, unit stride, tiles inside one depth slice (a row shift is then one uniform offset
  // of the whole tile), whole swizzle atoms per image row of the tile, the full K loop in one CTA
  const int kh_eff = ps ? 2 : d->kh;
  int yr_env = 1;
#ifdef EMO_CONV_DEBUG
  { const char* e = getenv("EMO_CONV_YREUSE"); if (e) yr_env = atoi(e); }  // instrumented build: per-tap form for the A/B tools
#endif
  const bool want_yreuse = yr_env != 0 && kh_eff > 1 && d->sh == 1 && d->sw == 1 && d->sd == 1 && p.td == 1 && p.tw >= 8 && ksplit == 1 && p.th + kh_eff - 1 <= 256;
  size_t ring_bytes = (size_t)(stages > kMaxStages ? kMaxStages : stages) * stage_bytes;
  if (want_yreuse) {
    // A ring of 2-3 halo tiles, the rest of the operand area as B ring (>= 3 tiles: one group's kh taps in flight)
    for (int KCy = KC0; KCy >= 32 && !p.yreuse; KCy >>= 1) {
      if (ps && KCy != 64) break;
      const size_t a_tile = (size_t)NP * p.tw * (p.th + kh_eff - 1) * KCy * 2, b_tile = (size_t)NP * BN * KCy * 2;
      if (2 * a_tile + 3 * b_tile > avail || (p.tw * KCy * 2) % 1024 != 0) continue;
      const int sa = (3 * a_tile + 4 * b_tile <= avail) ? 3 : 2;
      int sb = (int)((avail - sa * a_tile) / b_tile);
      if (sb > kMaxStages) sb = kMaxStages;
      p.yreuse = 1; p.sa = sa; p.sb = sb; p.a_rows = p.tw * (p.th + kh_eff - 1);
      KC = KCy;
      ring_bytes = sa * a_tile + sb * b_tile;
      stages = sb;
    }
  }
  p.kchunks = d->Cin / KC;
  if (stages > kMaxStages) stages = kMaxStages;
#ifdef EMO_CONV_DEBUG
  { const char* e = getenv("EMO_CONV_MAXSTAGES"); if (e && atoi(e) >= 2 && stages > atoi(e)) stages = atoi(e); }
#endif
  EMO_REQUIRE(stages >= 2, "emo_conv_igemm: tile does not fit shared memory (BN=%d KC=%d)", BN, KC);
  EMO_REQUIRE(!ps || KC == 64, "emo_conv_igemm: upconv tile does not fit with KC = 64");
  p.stages = stages;
  {
    // ~24 MMAs per accumulation chunk keeps the truncation bias of the tensor-core accumulator near 1e-6 relative; one-plane
    // operands: 16 MMAs = 256 channels of K (every MMA adds a full-size term: measured on an H100, 32 MMAs leave a bias of
    // -2.6e-6 relative, tests/test_fast_decoder_gpu.py)
    const int mmas_per_kstep = (KC / 16) * (NP == 3 ? 6 : NP == 2 ? 3 : 1);
    const int target = d->acc_chunk_mmas > 0 ? d->acc_chunk_mmas : (NP == 3 ? 24 : NP == 2 ? 48 : 16);
    p.flush = target / mmas_per_kstep < 1 ? 1 : target / mmas_per_kstep;
  }
  const size_t smem_bytes = ring_bytes + tail_bytes + 1024;
  const int total_tiles = p.m_tiles * p.n_tiles * p.ksplit;
  const int grid = total_tiles < sm_count ? total_tiles : sm_count;
  const long long per_n = (long long)d->Dout * d->Hout * d->Wout * d->Cout;
  const emo_apply_desc* post = d->post;
  if (ksplit > 1 && post && post->up == 1 && !d->out_nchw && !d->post_add && per_n <= (long long)kPostCluster * kPostThreads * kPostMaxV &&
      d->Cout <= kPostThreads && kPostThreads % d->Cout == 0 && (!post->stats || (post->G <= 64 && d->Cout % post->G == 0)))
    plan->finish = EMO_CONV_FINISH_POST;
  else if (ksplit > 1)
    plan->finish = post ? EMO_CONV_FINISH_FINALIZE_APPLY : EMO_CONV_FINISH_FINALIZE;
  else
    plan->finish = post ? EMO_CONV_FINISH_APPLY : EMO_CONV_FINISH_NONE;
  plan->NP = NP; plan->KC = KC; plan->f16 = f16; plan->ps = ps; plan->kh_eff = kh_eff;
  plan->kernel = -1;
  for (int k = 0; k < kNumConvKernels; ++k) {
    const ConvKernel& r = kConvKernels[k];
    if (r.NP == NP && r.f16 == (f16 != 0) && r.ps == (ps != 0) && r.KC == KC) plan->kernel = k;
  }
  EMO_REQUIRE(plan->kernel >= 0, "emo_conv_igemm: internal error: no kernel for NP=%d fp16=%d upconv=%d KC=%d", NP, f16, ps, KC);
  plan->grid = grid;
  // the per-CTA bias copy is placed after planning, above the planned area, where the opt-in maximum leaves room
  p.bias_smem = (d->bias && ksplit == 1 && p.ntc == 1 && smem_bytes + kMaxBN * sizeof(float) <= smem_limit) ? 1 : 0;
  plan->smem_bytes = smem_bytes + (p.bias_smem ? kMaxBN * sizeof(float) : 0);
  return EMO_OK;
}

}  // namespace emo

using namespace emo;

#ifdef EMO_CONV_DEBUG
extern "C" int emo_debug_conv_stamps(unsigned long long* host160x16) {
  return cudaMemcpyFromSymbol(host160x16, g_conv_stamps, sizeof(unsigned long long) * 160 * 16) == cudaSuccess ? 0 : -2;
}
// the phase clocks (g_conv_phase) into host160x8; reset != 0: zero them instead
extern "C" int emo_debug_conv_phases(unsigned long long* host160x8, int reset) {
  if (reset) {
    static const unsigned long long zeros[160 * 8] = {};
    return cudaMemcpyToSymbol(g_conv_phase, zeros, sizeof(zeros)) == cudaSuccess ? 0 : -2;
  }
  return cudaMemcpyFromSymbol(host160x8, g_conv_phase, sizeof(unsigned long long) * 160 * 8) == cudaSuccess ? 0 : -2;
}
#endif

extern "C" int emo_conv_plan(const emo_conv_desc* d, int sm_count, emo_conv_plan_info* out) {
  EMO_REQUIRE(out, "emo_conv_plan: null output");
  ConvPlan plan;
  const int rc = plan_conv(d, sm_count, &plan);
  if (rc) return rc;
  const ConvKParams& p = plan.p;
  memset(out, 0, sizeof(*out));
  out->kernel = plan.kernel; out->KC = plan.KC; out->NP = plan.NP; out->fp16 = plan.f16;
  out->BN = p.BN; out->ksplit = p.ksplit; out->yreuse = p.yreuse; out->sa = p.sa; out->sb = p.sb;
  out->stages = p.stages; out->flush = p.flush;
  out->tw = p.tw; out->th = p.th; out->td = p.td;
  out->m_tiles = p.m_tiles; out->n_tiles = p.n_tiles; out->grid = plan.grid; out->finish = plan.finish;
  return EMO_OK;
}

extern "C" int emo_conv_igemm(const emo_conv_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  int sm_count = 132, cur_dev = 0;
  {
    cudaGetDevice(&cur_dev);
    cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, cur_dev);
  }
  ConvPlan plan;
  {
    const int rc = plan_conv(d, sm_count, &plan);
    if (rc) return rc;
  }
  PFN_cuTensorMapEncodeTiled encode = get_encode();
  if (!encode) { set_error("emo_conv_igemm: cuTensorMapEncodeTiled entry point unavailable"); return EMO_ERR_CUDA; }
  const ConvKParams& p = plan.p;
  const int NP = plan.NP, KC = plan.KC, f16 = plan.f16, ps = plan.ps, kh_eff = plan.kh_eff, BN = p.BN, ksplit = p.ksplit;
  const int grid = plan.grid;
  const size_t smem_bytes = plan.smem_bytes;
  EMO_REQUIRE(smem_bytes <= 227 * 1024, "emo_conv_igemm: internal error: %zu bytes of shared memory", smem_bytes);

  // ---- tensor maps ----
  TMaps tm;
  memset(&tm, 0, sizeof(tm));
  {
    cuuint64_t gdim[5] = {(cuuint64_t)d->Cin, (cuuint64_t)d->Win, (cuuint64_t)d->Hin, (cuuint64_t)d->Din, (cuuint64_t)d->N};
    cuuint64_t gstr[4] = {(cuuint64_t)d->Cin * 2, (cuuint64_t)d->Win * d->Cin * 2, (cuuint64_t)d->Hin * d->Win * d->Cin * 2,
                          (cuuint64_t)d->Din * d->Hin * d->Win * d->Cin * 2};
    cuuint32_t box[5] = {(cuuint32_t)KC, (cuuint32_t)(p.tw * d->sw), (cuuint32_t)(p.yreuse ? p.th + kh_eff - 1 : p.th * d->sh), (cuuint32_t)(p.td * d->sd), 1};
    cuuint32_t estr[5] = {1, (cuuint32_t)d->sw, (cuuint32_t)d->sh, (cuuint32_t)d->sd, 1};
    const CUtensorMapSwizzle sw = (KC == 64) ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    const int taps = ps ? 16 : d->kd * d->kh * d->kw;  // sub-pixel mode: [4 phases][2x2 taps]
    cuuint64_t wdim[3] = {(cuuint64_t)d->Cin, (cuuint64_t)d->Cout_pad, (cuuint64_t)taps};
    cuuint64_t wstr[2] = {(cuuint64_t)d->Cin * 2, (cuuint64_t)d->Cout_pad * d->Cin * 2};
    cuuint32_t wbox[3] = {(cuuint32_t)KC, (cuuint32_t)BN, 1};
    cuuint32_t wes[3] = {1, 1, 1};
    const void* ap[3] = {d->a_hi, d->a_lo, d->a_lo2};
    const void* wp[3] = {d->w_hi, d->w_lo, d->w_lo2};
    const CUtensorMapDataType plane_type = f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    for (int pl = 0; pl < NP; ++pl) {
      EMO_REQUIRE(((uintptr_t)ap[pl] % 16) == 0 && ((uintptr_t)wp[pl] % 16) == 0, "emo_conv_igemm: planes must be 16-byte aligned");
      CUresult r1 = encode(&tm.a[pl], plane_type, 5, (void*)ap[pl], gdim, gstr, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      CUresult r2 = encode(&tm.b[pl], plane_type, 3, (void*)wp[pl], wdim, wstr, wbox, wes,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r1 != CUDA_SUCCESS || r2 != CUDA_SUCCESS) {
        set_error("emo_conv_igemm: cuTensorMapEncodeTiled failed: A %d W %d (Cin=%d W=%d H=%d D=%d N=%d box=%d,%d,%d BN=%d)", (int)r1,
                  (int)r2, d->Cin, d->Win, d->Hin, d->Din, d->N, p.tw, p.th, p.td, BN);
        return EMO_ERR_CUDA;
      }
    }
  }

  const auto kernel = kConvKernels[plan.kernel].fn;
  static bool attr_set[kNumConvKernels][64] = {};  // the opt-in is per function AND per device (227 KB covers every configuration)
  cudaError_t e;
  if (!attr_set[plan.kernel][cur_dev & 63]) {
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) { set_error("emo_conv_igemm: smem attribute: %s", cudaGetErrorString(e)); return EMO_ERR_CUDA; }
    attr_set[plan.kernel][cur_dev & 63] = true;
  }
  kernel<<<grid, kThreads, smem_bytes, stream>>>(tm, p);
  e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("emo_conv_igemm: launch: %s", cudaGetErrorString(e)); return EMO_ERR_CUDA; }
  const emo_apply_desc* post = d->post;
  if (plan.finish == EMO_CONV_FINISH_POST) {
    // small split-K layer with a post-op: one cluster per sample finishes the convolution, normalises, activates and writes the
    // next convolution's operand planes (splitk_post_kernel)
    PostParams f;
    memset(&f, 0, sizeof(f));
    f.ws = d->splitk_ws; f.ksplit = ksplit; f.part_elems = p.ws_part_elems;
    f.N = d->N; f.C = d->Cout; f.S = (long long)d->Dout * d->Hout * d->Wout;
    f.bias = d->bias; f.residual = d->residual; f.conv_act = d->act;
    f.ap = *post;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)(kPostCluster * d->N));
    cfg.blockDim = dim3(kPostThreads);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = kPostCluster; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    e = cudaLaunchKernelEx(&cfg, splitk_post_kernel, f);
    if (e != cudaSuccess) { set_error("emo_conv_igemm: post launch: %s", cudaGetErrorString(e)); return EMO_ERR_CUDA; }
    return check_launch("emo_conv_igemm");
  }
  if (ksplit > 1) {
    FinParams f;
    f.ws = d->splitk_ws; f.ksplit = ksplit; f.part_elems = p.ws_part_elems; f.out = d->out; f.N = d->N; f.C = d->Cout;
    f.S = (long long)d->Dout * d->Hout * d->Wout;
    f.bias = d->bias; f.residual = d->residual; f.post_add = d->post_add; f.act = d->act; f.out_nchw = d->out_nchw;
    f.stats = d->stats; f.G = d->G;
    long long bx = cdivll(f.S * f.C, 256 * 2);
    if (bx > sm_count * 4ll) bx = sm_count * 4ll;
    if (bx < 1) bx = 1;
    dim3 fg((unsigned)bx, (unsigned)d->N);
    launch_kernel(splitk_finalize_kernel, fg, 256, d->stats ? 2 * d->G * sizeof(double) : 0, stream, f);
  }
  if (post) {
    // every other layer: the post-op is the ordinary elementwise pass over the convolution's output
    int rc = check_launch("emo_conv_igemm");
    if (rc) return rc;
    emo_apply_desc ap = *post;
    ap.x = d->out;
    return emo_apply(&ap, stream_);
  }
  return check_launch("emo_conv_igemm");
}
