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
  int dbg;    // EMO_CONV_DEBUG builds only (tools/conv_bound_probe.py): 1 skip TMA loads, 2 skip MMAs.  Results are garbage;
              // only the timing is of interest.
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
  // sub-pixel mode (conv_igemm_ps_kernel): 3x3 conv over the nearest-x2 upsampling of the input, evaluated on the LOW-resolution
  // planes.  Dout/Hout/Wout above then describe the low-resolution pixel grid the tiles walk; the output tensor is
  // [N][Dout][oH = 2 Hout][oW = 2 Wout][Cout].  The N-tile index carries the output phase: nt = phase * ntc + channel tile,
  // phase = 2 * (row parity) + (column parity); each phase has its own four 2x2 taps (weights [phase * 4 + tap]).
  int oH, oW;
  int ntc;  // channel tiles per phase (= Cout_pad / BN)
  float out_scale;  // conv_igemm_f16_kernel: 1 / (activation plane scale * weight plane scale)
  // row-reuse mode (stride-1 convolutions with kh > 1 on tiles of one depth slice): the A operand of a (kernel column,
  // k-chunk) group is ONE halo tile of a_rows = tw * (th + kh - 1) pixels serving all kh tap rows; A ring of `sa` halo tiles,
  // B ring of `sb` weight tiles (see the kernel's producer role)
  int yreuse, sa, sb, a_rows;
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
#else
#define EMO_STAMP(k, cond) do { } while (0)
#endif

struct TMaps {
  CUtensorMap a[3];  // activation planes: hi, lo, lo2
  CUtensorMap b[3];  // weight planes
};

#define EMO_CONV_PS 0
#define EMO_CONV_F16 0
#define EMO_CONV_KERNEL_NAME conv_igemm_kernel
#include "conv_igemm_kernel.inc"
#undef EMO_CONV_PS
#undef EMO_CONV_KERNEL_NAME
#define EMO_CONV_PS 1
#define EMO_CONV_KERNEL_NAME conv_igemm_ps_kernel
#include "conv_igemm_kernel.inc"
#undef EMO_CONV_PS
#undef EMO_CONV_F16
#undef EMO_CONV_KERNEL_NAME
#define EMO_CONV_PS 0
#define EMO_CONV_F16 1
#define EMO_CONV_KERNEL_NAME conv_igemm_f16_kernel
#include "conv_igemm_kernel.inc"
#undef EMO_CONV_PS
#undef EMO_CONV_KERNEL_NAME
#define EMO_CONV_PS 1
#define EMO_CONV_KERNEL_NAME conv_igemm_ps_f16_kernel
#include "conv_igemm_kernel.inc"
#undef EMO_CONV_PS
#undef EMO_CONV_F16
#undef EMO_CONV_KERNEL_NAME

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
  plan->kernel = NP == 1 ? (ps ? EMO_CONV_KERNEL_H1_UPCONV_KC64 : KC == 64 ? EMO_CONV_KERNEL_H1_KC64 : EMO_CONV_KERNEL_H1_KC32)
                 : f16 ? (KC == 64 ? EMO_CONV_KERNEL_F16_KC64 : EMO_CONV_KERNEL_F16_KC32)
                 : ps ? EMO_CONV_KERNEL_UPCONV_KC64
                 : NP == 3 ? (KC == 64 ? EMO_CONV_KERNEL_BF16X3_KC64 : EMO_CONV_KERNEL_BF16X3_KC32)
                           : (KC == 64 ? EMO_CONV_KERNEL_BF16X2_KC64 : EMO_CONV_KERNEL_BF16X2_KC32);
  plan->grid = grid;
  plan->smem_bytes = smem_bytes;
  return EMO_OK;
}

}  // namespace emo

using namespace emo;

#ifdef EMO_CONV_DEBUG
extern "C" int emo_debug_conv_stamps(unsigned long long* host160x16) {
  return cudaMemcpyFromSymbol(host160x16, g_conv_stamps, sizeof(unsigned long long) * 160 * 16) == cudaSuccess ? 0 : -2;
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

  cudaError_t e;
#define EMO_LAUNCH_CONV(KERNEL_, KC_, NP_)                                                                                 \
  do {                                                                                                                    \
    static bool attr_set_dev[64] = {false}; /* the opt-in is per function AND per device (227 KB covers every configuration) */ \
    bool& attr_set = attr_set_dev[cur_dev & 63];                                                                          \
    if (!attr_set) {                                                                                                      \
      e = cudaFuncSetAttribute(KERNEL_<KC_, NP_>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);               \
      if (e != cudaSuccess) { set_error("emo_conv_igemm: smem attribute: %s", cudaGetErrorString(e)); return EMO_ERR_CUDA; } \
      attr_set = true;                                                                                                    \
    }                                                                                                                     \
    KERNEL_<KC_, NP_><<<grid, kThreads, smem_bytes, stream>>>(tm, p);                                                     \
    e = cudaGetLastError();                                                                                               \
    if (e != cudaSuccess) { set_error("emo_conv_igemm: launch: %s", cudaGetErrorString(e)); return EMO_ERR_CUDA; }         \
  } while (0)
  if (NP == 1) {
    if (ps) EMO_LAUNCH_CONV(conv_igemm_ps_f16_kernel, 64, 1);
    else if (KC == 64) EMO_LAUNCH_CONV(conv_igemm_f16_kernel, 64, 1);
    else EMO_LAUNCH_CONV(conv_igemm_f16_kernel, 32, 1);
  } else if (f16) {
    if (KC == 64) EMO_LAUNCH_CONV(conv_igemm_f16_kernel, 64, 2);
    else EMO_LAUNCH_CONV(conv_igemm_f16_kernel, 32, 2);
  } else if (ps) {
    EMO_LAUNCH_CONV(conv_igemm_ps_kernel, 64, 2);
  } else if (NP == 3) {
    if (KC == 64) EMO_LAUNCH_CONV(conv_igemm_kernel, 64, 3);
    else EMO_LAUNCH_CONV(conv_igemm_kernel, 32, 3);
  } else {
    if (KC == 64) EMO_LAUNCH_CONV(conv_igemm_kernel, 64, 2);
    else EMO_LAUNCH_CONV(conv_igemm_kernel, 32, 2);
  }
#undef EMO_LAUNCH_CONV
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
