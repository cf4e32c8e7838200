// GroupNorm statistics / affine finalisation / fused apply (HBM-bound elementwise passes).
//
// nn.GroupNorm(32, C, eps=1e-5)  networks/volumetric_avatar/utils.py:953,957
// AdaptiveGroupNorm              utils.py:302-325 (+ assign_adaptive_norm_params :983-995):
//     y = (GN(x)*w + b) * (w + dw) + (b + db)
// ResBlock pre-activation order  utils.py:761-788: [nearest up] -> norm -> ReLU -> conv
// The apply pass writes what the next tensor-core conv consumes: bf16 (hi, lo) planes, channels-last.
#include <stdlib.h>

#include "common.cuh"

namespace emo {

// ---- statistics: x [N][S][C] fp32, per (n, g) sum and sum of squares, double accumulation across CTAs ----
__global__ void __launch_bounds__(256) gn_stats_kernel(const float* __restrict__ x, int N, long long S, int C, int G,
                                                       double* __restrict__ stats, int chunks) {
  // grid = N * chunks; each CTA reduces a slab of spatial positions for all channels
  const int n = blockIdx.x / chunks, ch = blockIdx.x % chunks;
  const long long s_per = (S + chunks - 1) / chunks;
  const long long s0 = (long long)ch * s_per;
  const long long s1 = (s0 + s_per < S) ? s0 + s_per : S;
  const int cpg = C / G;
  extern __shared__ double sh[];  // [2][G]; fp64: sums of fp32 values are exact, so the result does not depend on the order of the atomics
  for (int i = threadIdx.x; i < 2 * G; i += blockDim.x) sh[i] = 0.0;
  __syncthreads();
  const int c4n = C >> 2;
  const float4* x4 = (const float4*)(x + (long long)n * S * C);
  // each thread owns one float4 channel slot (c4) and a row slot; accumulates in registers, flushes once
  const int L = c4n < (int)blockDim.x ? c4n : (int)blockDim.x;
  const int rpi = blockDim.x / L;  // rows handled per pass
  const int rslot = threadIdx.x / L;
  if (rslot < rpi) {
    for (int c4 = threadIdx.x % L; c4 < c4n; c4 += L) {
      float acc_s[4] = {0, 0, 0, 0}, acc_q[4] = {0, 0, 0, 0};
      for (long long s = s0 + rslot; s < s1; s += rpi) {
        const float4 v = __ldg(x4 + s * c4n + c4);
        acc_s[0] += v.x; acc_q[0] = fmaf(v.x, v.x, acc_q[0]);
        acc_s[1] += v.y; acc_q[1] = fmaf(v.y, v.y, acc_q[1]);
        acc_s[2] += v.z; acc_q[2] = fmaf(v.z, v.z, acc_q[2]);
        acc_s[3] += v.w; acc_q[3] = fmaf(v.w, v.w, acc_q[3]);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int g = (c4 * 4 + j) / cpg;
        atomicAdd(&sh[g], (double)acc_s[j]);
        atomicAdd(&sh[G + g], (double)acc_q[j]);
      }
    }
  }
  __syncthreads();
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    atomicAdd(&stats[((long long)n * G + g) * 2], sh[g]);
    atomicAdd(&stats[((long long)n * G + g) * 2 + 1], sh[G + g]);
  }
}

// ---- finalize: stats -> per-(n,c) scale/shift ----
__global__ void gn_finalize_kernel(const emo_gn_finalize_desc d) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= d.N * d.C) return;
  const int n = idx / d.C, c = idx % d.C;
  const int g = c / (d.C / d.G);
  const double s = d.stats[((long long)n * d.G + g) * 2], q = d.stats[((long long)n * d.G + g) * 2 + 1];
  const double mean = s / d.count;
  double var = q / d.count - mean * mean;
  if (var < 0) var = 0;
  const float rstd = (float)(1.0 / sqrt(var + (double)d.eps));
  float gam = d.gamma ? d.gamma[c] : 1.f, bet = d.beta ? d.beta[c] : 0.f;
  if (d.ada_w) {
    const float aw = d.ada_w[idx], ab = d.ada_b[idx];
    bet = bet * aw + ab;
    gam = gam * aw;
  }
  const float A = rstd * gam;
  d.A[idx] = A;
  d.B[idx] = bet - (float)mean * A;
}

// resident CTAs per SM the apply kernels are compiled for (register cap 65536 / (256 * n)).  Measured round 2 (tools/apply_probe.py,
// 512^2 x 128): 4 -> 56.1 us, 6 (40 registers, ~100 B of spills) -> 60.1 us; unconstrained (66 registers, 3 CTAs) was 1 % of the frame slower.
#ifndef EMO_APPLY_MIN_CTAS
#define EMO_APPLY_MIN_CTAS 4
#endif
#define EMO_APPLY_F16 0
#define EMO_APPLY_KERNEL_NAME apply_kernel
#include "apply_kernel.inc"
#undef EMO_APPLY_F16
#undef EMO_APPLY_KERNEL_NAME
#define EMO_APPLY_F16 1
#define EMO_APPLY_KERNEL_NAME apply_f16_kernel
#include "apply_kernel.inc"
#undef EMO_APPLY_F16
#undef EMO_APPLY_KERNEL_NAME

// Image head (emo_gn_head): one warp handles 8 pixels per step.  Lane l owns channels 4l..4l+3 (+128k): a warp load reads a
// pixel's whole channel vector (512 B at C = 128); the 8 x 4 per-lane partial dot products are transpose-reduced over the
// warp with 31 shuffles, after which lane l = 4u + o holds output o of pixel u.
__global__ void __launch_bounds__(256) gn_head_kernel(const emo_gn_head_desc d) {
  extern __shared__ float sAB[];  // A[C], B[C] of this CTA's sample, then w[4][C] (rows >= Cout are zero)
  const int n = blockIdx.y;
  const int C = d.C;
  float* sW = sAB + 2 * C;
  {
    const int cpg = C / d.G;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      const int g = c / cpg;
      const double s = d.stats[((long long)n * d.G + g) * 2], q = d.stats[((long long)n * d.G + g) * 2 + 1];
      const double mean = s / d.count;
      double var = q / d.count - mean * mean;
      if (var < 0) var = 0;
      const float rstd = (float)(1.0 / sqrt(var + (double)d.eps));
      const float A = rstd * d.gamma[c];
      sAB[c] = A;
      sAB[C + c] = d.beta[c] - (float)mean * A;
      for (int o = 0; o < 4; ++o) sW[o * C + c] = o < d.Cout ? d.w[(long long)o * C + c] : 0.f;
    }
    __syncthreads();
  }
  const int lane = threadIdx.x & 31;
  const int warps_per_grid = gridDim.x * (blockDim.x >> 5);
  const int warp_id = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long S = d.S;
  const float* xn = d.x + (long long)n * S * C;
  float bo = 0.f;
  if (d.bias && (lane & 3) < d.Cout) bo = d.bias[lane & 3];
  for (long long p0 = (long long)warp_id * 8; p0 < S; p0 += (long long)warps_per_grid * 8) {
    float val[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) val[i] = 0.f;
    for (int c = 4 * lane; c < C; c += 128) {
      float4 v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u)
        v[u] = (p0 + u < S) ? __ldg((const float4*)(xn + (p0 + u) * C + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float4 a = *(const float4*)&sAB[c];
      const float4 b = *(const float4*)&sAB[C + c];
      float4 w[4];
#pragma unroll
      for (int o = 0; o < 4; ++o) w[o] = *(const float4*)&sW[o * C + c];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const float y0 = fmaxf(fmaf(v[u].x, a.x, b.x), 0.f), y1 = fmaxf(fmaf(v[u].y, a.y, b.y), 0.f);
        const float y2 = fmaxf(fmaf(v[u].z, a.z, b.z), 0.f), y3 = fmaxf(fmaf(v[u].w, a.w, b.w), 0.f);
#pragma unroll
        for (int o = 0; o < 4; ++o)
          val[u * 4 + o] += y0 * w[o].x + y1 * w[o].y + y2 * w[o].z + y3 * w[o].w;
      }
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
      const bool upper = (lane & off) != 0;
#pragma unroll
      for (int j = 0; j < off; ++j) {
        const float send = upper ? val[j] : val[j + off];
        const float keep = upper ? val[j + off] : val[j];
        val[j] = keep + __shfl_xor_sync(0xffffffffu, send, off);
      }
    }
    const int u = lane >> 2, o = lane & 3;
    if (o < d.Cout && p0 + u < S) d.out[((long long)n * d.Cout + o) * S + p0 + u] = act_apply(val[0] + bo, d.act_out);
  }
}

__global__ void split_kernel(const float* __restrict__ x, long long n4, uint2* __restrict__ hi, uint2* __restrict__ lo,
                             uint2* __restrict__ lo2) {
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n4; t += (long long)gridDim.x * blockDim.x) {
    uint2 h, l, l2;
    if (lo2) {
      split4x3(__ldg((const float4*)x + t), h, l, l2);
      lo2[t] = l2;
    } else {
      split4(__ldg((const float4*)x + t), h, l);
    }
    hi[t] = h; lo[t] = l;
  }
}

__global__ void split_f16_kernel(const float* __restrict__ x, long long n4, float scale, uint2* __restrict__ hi, uint2* __restrict__ lo) {
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n4; t += (long long)gridDim.x * blockDim.x) {
    const float4 v = __ldg((const float4*)x + t);
    if (lo) {
      uint2 h, l;
      split4_h(v, scale, h, l);
      hi[t] = h; lo[t] = l;
    } else {
      hi[t] = plane4_h(v, scale);
    }
  }
}

__global__ void flush_kernel(float4* buf, long long n4) {
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n4; t += (long long)gridDim.x * blockDim.x)
    buf[t] = make_float4(0.f, 0.f, 0.f, 0.f);
}
// read the flush buffer back: the dirty lines the write pass left in L2 are written out and replaced by CLEAN lines of the
// same buffer, so that the kernel under test does not pay for write-backs of the flush itself
__global__ void flush_read_kernel(const float4* buf, long long n4, float* sink) {
  float acc = 0.f;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n4; t += (long long)gridDim.x * blockDim.x) {
    const float4 v = __ldcg(buf + t);
    acc += v.x + v.y + v.z + v.w;
  }
  if (acc == 123.456f) *sink = acc;  // never true (the buffer holds zeros): keeps the loads alive
}

}  // namespace emo

using namespace emo;

extern "C" int emo_gn_stats(const float* x, int N, long long spatial, int C, int G, double* stats, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(x && stats, "emo_gn_stats: null pointer");
  EMO_REQUIRE(C % 4 == 0 && G > 0 && C % G == 0, "emo_gn_stats: C=%d must be a multiple of 4 and of G=%d", C, G);
  EMO_REQUIRE(((uintptr_t)x % 16) == 0, "emo_gn_stats: x must be 16-byte aligned");
  long long work = spatial * (C / 4);
  int chunks = (int)(work / (256 * 16));
  if (chunks < 1) chunks = 1;
  const int max_chunks = (132 * 8) / (N > 0 ? N : 1) > 0 ? (132 * 8) / N : 1;
  if (chunks > max_chunks) chunks = max_chunks;
  launch_kernel(gn_stats_kernel, N * chunks, 256, 2 * G * sizeof(double), stream, x, N, spatial, C, G, stats, chunks);
  return check_launch("emo_gn_stats");
}

extern "C" int emo_gn_finalize(const emo_gn_finalize_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(d && d->stats && d->A && d->B, "emo_gn_finalize: null pointer");
  EMO_REQUIRE(d->G > 0 && d->C % d->G == 0, "emo_gn_finalize: C=%d not divisible by G=%d", d->C, d->G);
  EMO_REQUIRE((d->ada_w == nullptr) == (d->ada_b == nullptr), "emo_gn_finalize: ada_w/ada_b must come together");
  const int total = d->N * d->C;
  launch_kernel(gn_finalize_kernel, cdiv(total, 128), 128, 0, stream, *d);
  return check_launch("emo_gn_finalize");
}

extern "C" int emo_apply(const emo_apply_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(d && d->x, "emo_apply: null input");
  EMO_REQUIRE(d->out || (d->out_hi && (d->out_lo || d->plane_fp16)), "emo_apply: no output");
  EMO_REQUIRE((!d->out_lo || d->out_hi) && (!d->out_hi || d->out_lo || d->plane_fp16),
              "emo_apply: operand planes are out_hi + out_lo, or out_hi alone with plane_fp16");
  EMO_REQUIRE(d->C % 4 == 0, "emo_apply: C=%d must be a multiple of 4", d->C);
  EMO_REQUIRE(d->up == 1 || d->up == 2, "emo_apply: up must be 1 or 2");
  EMO_REQUIRE((d->A == nullptr) == (d->B == nullptr) && (d->A2 == nullptr) == (d->B2 == nullptr), "emo_apply: A/B must come in pairs");
  if (d->stats) EMO_REQUIRE(d->G > 0 && d->C % d->G == 0 && d->count > 0, "emo_apply: bad GroupNorm arguments");
  // V = 2 (two consecutive float4 per thread, 16-byte plane stores) whenever C % 8 == 0; one float4 per thread otherwise
  // (measured round 2: forcing V = 1 everywhere costs 3% of the frame)
  const int V = (d->C % 8 == 0) ? 2 : 1;
  const long long per_n = (long long)d->D * d->H * d->W * (d->C / (4 * V));
  long long blocks = cdivll(per_n, 256);
  const long long cap = (132ll * 32) / (d->N > 0 ? d->N : 1);
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  const dim3 grid((unsigned)blocks, (unsigned)d->N);
  const size_t smem = d->stats ? 2 * (size_t)d->C * sizeof(float) : 0;
  EMO_REQUIRE(smem <= 48 * 1024, "emo_apply: C=%d too large for the fused finalisation", d->C);
  if (d->plane_fp16) {
    EMO_REQUIRE(!d->out_lo2 && d->plane_scale > 0.f, "emo_apply: fp16 planes are one or two (no out_lo2) and need a positive plane_scale");
    if (d->up == 1 && V == 2) launch_kernel(apply_f16_kernel<1, 2>, grid, 256, smem, stream, *d);
    else if (d->up == 1) launch_kernel(apply_f16_kernel<1, 1>, grid, 256, smem, stream, *d);
    else if (V == 2) launch_kernel(apply_f16_kernel<2, 2>, grid, 256, smem, stream, *d);
    else launch_kernel(apply_f16_kernel<2, 1>, grid, 256, smem, stream, *d);
    return check_launch("emo_apply");
  }
  if (d->up == 1 && V == 2) launch_kernel(apply_kernel<1, 2>, grid, 256, smem, stream, *d);
  else if (d->up == 1) launch_kernel(apply_kernel<1, 1>, grid, 256, smem, stream, *d);
  else if (V == 2) launch_kernel(apply_kernel<2, 2>, grid, 256, smem, stream, *d);
  else launch_kernel(apply_kernel<2, 1>, grid, 256, smem, stream, *d);
  return check_launch("emo_apply");
}

extern "C" int emo_gn_head(const emo_gn_head_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(d && d->x && d->stats && d->gamma && d->beta && d->w && d->out, "emo_gn_head: null pointer");
  EMO_REQUIRE(d->Cout >= 1 && d->Cout <= 4, "emo_gn_head: Cout=%d must be 1..4", d->Cout);
  EMO_REQUIRE(d->C % 4 == 0 && d->G > 0 && d->C % d->G == 0, "emo_gn_head: C=%d must be a multiple of 4 and of G=%d", d->C, d->G);
  EMO_REQUIRE(((uintptr_t)d->x % 16) == 0, "emo_gn_head: x must be 16-byte aligned");
  if (d->N == 0 || d->S == 0) return EMO_OK;
  const size_t smem = 6 * (size_t)d->C * sizeof(float);
  EMO_REQUIRE(smem <= 48 * 1024, "emo_gn_head: C=%d too large", d->C);
  long long blocks = cdivll(d->S, 8 * 8);  // 8 warps x 8 pixels per step
  if (blocks > 132 * 8) blocks = 132 * 8;
  if (blocks < 1) blocks = 1;
  launch_kernel(gn_head_kernel, dim3((unsigned)blocks, (unsigned)d->N), 256, smem, stream, *d);
  return check_launch("emo_gn_head");
}

extern "C" int emo_split_bf16(const float* x, long long n, void* hi, void* lo, void* lo2, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(x && hi && lo, "emo_split_bf16: null pointer");
  EMO_REQUIRE(n % 4 == 0, "emo_split_bf16: n must be a multiple of 4");
  long long blocks = cdivll(n / 4, 256);
  if (blocks > 132ll * 32) blocks = 132ll * 32;
  if (blocks < 1) blocks = 1;
  launch_kernel(split_kernel, (unsigned)blocks, 256, 0, stream, x, n / 4, (uint2*)hi, (uint2*)lo, (uint2*)lo2);
  return check_launch("emo_split_bf16");
}

extern "C" int emo_split_f16(const float* x, long long n, float scale, void* hi, void* lo, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(x && hi, "emo_split_f16: null pointer");
  EMO_REQUIRE(n % 4 == 0 && scale > 0.f, "emo_split_f16: n must be a multiple of 4 and scale positive");
  long long blocks = cdivll(n / 4, 256);
  if (blocks > 132ll * 32) blocks = 132ll * 32;
  if (blocks < 1) blocks = 1;
  launch_kernel(split_f16_kernel, (unsigned)blocks, 256, 0, stream, x, n / 4, scale, (uint2*)hi, (uint2*)lo);
  return check_launch("emo_split_f16");
}

extern "C" int emo_l2_flush(void* buf, long long bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(buf && bytes >= 16, "emo_l2_flush: bad buffer");
  launch_kernel(flush_kernel, 132 * 8, 256, 0, stream, (float4*)buf, bytes / 16);
  return check_launch("emo_l2_flush");
}

extern "C" int emo_l2_flush_clean(void* buf, long long bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(buf && bytes >= 32, "emo_l2_flush_clean: bad buffer");
  launch_kernel(flush_kernel, 132 * 8, 256, 0, stream, (float4*)buf, bytes / 16);
  launch_kernel(flush_read_kernel, 132 * 8, 256, 0, stream, (const float4*)buf, bytes / 16, (float*)buf);
  return check_launch("emo_l2_flush_clean");
}
