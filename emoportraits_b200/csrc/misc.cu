// Small dense ops (fp32 SIMT, exact): linear layers, the RGB stem convolutions, resampling, pose algebra.
#include "common.cuh"
#include "pose_math.cuh"

#include <stdarg.h>
#include <stdlib.h>

namespace emo {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return EMO_ERR_CUDA;
  }
  return EMO_OK;
}

// ------------------------------------------------------------------------------------------------
// linear: one warp per output element (m, n), lanes stride over K.  Sizes are tiny (<= 20 MFLOP).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) linear_kernel(const emo_linear_desc d) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= d.M * d.N) return;
  const int m = warp / d.N, n = warp % d.N;
  const float* xr = d.x + (long long)m * d.xs_m;
  const float* wr = d.w + (long long)n * d.K;
  float acc = 0.f;
  for (int k = lane; k < d.K; k += 32) acc = fmaf(__ldg(xr + (long long)k * d.xs_k), __ldg(wr + k), acc);
  acc = warp_sum(acc);
  if (lane == 0) {
    const long long o = (long long)m * d.os_m + (long long)n * d.os_n;
    if (d.bias) acc += d.bias[n];
    if (d.add) acc += d.add[o];
    d.out[o] = act_apply(acc * d.scale, d.act);
  }
}

// ------------------------------------------------------------------------------------------------
// direct conv, channels-last, tiny Cin (RGB stems).  Thread = (pixel, 4 output channels).
// weights [kh][kw][Cin_pad][Cout]: the co-vector load is coalesced across the co-threads of a pixel,
// the activation load is a warp broadcast.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) conv_direct_kernel(const emo_conv_direct_desc d) {
  const int co4n = d.Cout >> 2;
  const long long total = (long long)d.N * d.Hout * d.Wout * co4n;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  extern __shared__ double sstat[];  // [2][G] when stats requested
  if (d.stats) {
    for (int i = threadIdx.x; i < 2 * d.G; i += blockDim.x) sstat[i] = 0.0;
    __syncthreads();
  }
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  int co4 = 0, n = 0;
  const bool active = t < total;
  if (active) {
    co4 = (int)(t % co4n);
    long long pix = t / co4n;
    const int ow = (int)(pix % d.Wout); pix /= d.Wout;
    const int oh = (int)(pix % d.Hout); pix /= d.Hout;
    n = (int)pix;
    if (d.bias) acc = __ldg((const float4*)d.bias + co4);
    for (int ky = 0; ky < d.kh; ++ky) {
      const int iy = oh * d.stride + ky - d.pad;
      if (iy < 0 || iy >= d.Hin) continue;
      for (int kx = 0; kx < d.kw; ++kx) {
        const int ix = ow * d.stride + kx - d.pad;
        if (ix < 0 || ix >= d.Win) continue;
        const float* xp = d.x + (((long long)n * d.Hin + iy) * d.Win + ix) * d.Cin_pad;
        const float4* wp = (const float4*)(d.w + ((long long)(ky * d.kw + kx) * d.Cin_pad) * d.Cout) + co4;
        for (int ci = 0; ci < d.Cin_pad; ++ci) {
          const float xv = __ldg(xp + ci);
          const float4 wv = __ldg(wp + (long long)ci * co4n);
          acc.x = fmaf(xv, wv.x, acc.x); acc.y = fmaf(xv, wv.y, acc.y);
          acc.z = fmaf(xv, wv.z, acc.z); acc.w = fmaf(xv, wv.w, acc.w);
        }
      }
    }
    ((float4*)d.out)[t] = acc;
  }
  if (d.stats) {
    // a CTA may straddle two samples only if Hout*Wout*co4n < blockDim; host guarantees divisibility instead
    if (active) {
      const int cpg = d.Cout / d.G;
      const float a[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int g = (co4 * 4 + j) / cpg;
        atomicAdd(&sstat[g], (double)a[j]);
        atomicAdd(&sstat[d.G + g], (double)(a[j] * a[j]));
      }
    }
    __syncthreads();
    const long long first = (long long)blockIdx.x * blockDim.x;
    const int nb = (int)(first / ((long long)d.Hout * d.Wout * co4n));
    for (int g = threadIdx.x; g < d.G; g += blockDim.x) {
      atomicAdd(&d.stats[((long long)nb * d.G + g) * 2], sstat[g]);
      atomicAdd(&d.stats[((long long)nb * d.G + g) * 2 + 1], sstat[d.G + g]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// RGB stem operand for the tensor cores: thread = one pixel.  Its 7 horizontal taps (float4 each, neighbouring threads read
// overlapping taps through L1) become 28 fp16 channels of (value * scale), then 4 zero channels: 64 bytes, 4 x 16-byte stores.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) stem_pack_kernel(const float4* __restrict__ x, int H, int W, long long pixels, float s,
                                                       uint4* __restrict__ out) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < pixels; p += (long long)gridDim.x * blockDim.x) {
    const int w = (int)(p % W);
    uint2 v[8];
#pragma unroll
    for (int kx = 0; kx < 7; ++kx) {
      const int ix = w + kx - 3;
      v[kx] = (ix >= 0 && ix < W) ? plane4_h(__ldg(x + p + (kx - 3)), s) : make_uint2(0u, 0u);
    }
    v[7] = make_uint2(0u, 0u);
    uint4* o = out + p * 4;
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = make_uint4(v[2 * j].x, v[2 * j].y, v[2 * j + 1].x, v[2 * j + 1].y);
  }
}

// ------------------------------------------------------------------------------------------------
// trilinear upsample (align_corners=False), factors in {1,2} per axis, channels-last, optional add + GN stats
//   src = max((dst + 0.5)/f - 0.5, 0); i0 = floor(src); i1 = min(i0+1, n-1); l = src - i0
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void up_coord(int o, int f, int n_in, int& i0, int& i1, float& l) {
  if (f == 1) { i0 = o; i1 = o; l = 0.f; return; }
  float s = ((float)o + 0.5f) * 0.5f - 0.5f;
  s = fmaxf(s, 0.f);
  i0 = (int)s;
  i1 = i0 + (i0 < n_in - 1 ? 1 : 0);
  l = s - (float)i0;
}

__global__ void __launch_bounds__(256) upsample_trilinear_kernel(const emo_resample_desc d) {
  const int c4n = d.C >> 2;
  const int Do = d.D * d.fd, Ho = d.H * d.fh, Wo = d.W * d.fw;
  const long long So = (long long)Do * Ho * Wo;
  const long long per_n = So * c4n;
  // grid.y = sample index so that a CTA never straddles samples (needed for the stats reduction)
  const int n = blockIdx.y;
  extern __shared__ double sstat[];
  if (d.stats) {
    for (int i = threadIdx.x; i < 2 * d.G; i += blockDim.x) sstat[i] = 0.0;
    __syncthreads();
  }
  const float4* x4 = (const float4*)d.x + (long long)n * d.D * d.H * d.W * c4n;
  // statistics: when the grid stride is a multiple of the channel-slot count a thread owns ONE slot for its whole loop and sums
  // it in registers (one shared-memory atomic per thread and channel instead of one per element: the per-element form made
  // the 32 x 64 x 64 x 64 upsample of the warp generator run at 1 TB/s)
  const bool fixed_c = ((long long)gridDim.x * blockDim.x) % c4n == 0;
  float rs[4] = {0.f, 0.f, 0.f, 0.f}, rq[4] = {0.f, 0.f, 0.f, 0.f};
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < per_n; t += (long long)gridDim.x * blockDim.x) {
    // 32-bit index arithmetic (the host requires per_n < 2^31): the 64-bit form is four emulated divisions per float4
    const unsigned tu = (unsigned)t;
    const int c4 = (int)(tu % (unsigned)c4n);
    unsigned s = tu / (unsigned)c4n;
    const int ow = (int)(s % (unsigned)Wo); s /= (unsigned)Wo;
    const int oh = (int)(s % (unsigned)Ho); s /= (unsigned)Ho;
    const int od = (int)s;
    int z0, z1, y0, y1, x0, x1;
    float lz, ly, lx;
    up_coord(od, d.fd, d.D, z0, z1, lz);
    up_coord(oh, d.fh, d.H, y0, y1, ly);
    up_coord(ow, d.fw, d.W, x0, x1, lx);
    auto ld = [&](int z, int y, int x) { return __ldg(x4 + (((long long)z * d.H + y) * d.W + x) * c4n + c4); };
    const float hz = 1.f - lz, hy = 1.f - ly, hx = 1.f - lx;
    float4 acc;
    {
      const float4 a000 = ld(z0, y0, x0), a001 = ld(z0, y0, x1), a010 = ld(z0, y1, x0), a011 = ld(z0, y1, x1);
      const float4 a100 = ld(z1, y0, x0), a101 = ld(z1, y0, x1), a110 = ld(z1, y1, x0), a111 = ld(z1, y1, x1);
#define EMO_TRI(f) \
  (hz * (hy * (hx * a000.f + lx * a001.f) + ly * (hx * a010.f + lx * a011.f)) + \
   lz * (hy * (hx * a100.f + lx * a101.f) + ly * (hx * a110.f + lx * a111.f)))
      acc.x = EMO_TRI(x); acc.y = EMO_TRI(y); acc.z = EMO_TRI(z); acc.w = EMO_TRI(w);
#undef EMO_TRI
    }
    const long long o = (long long)n * per_n + t;
    if (d.add) {
      const float4 a = __ldg((const float4*)d.add + o);
      acc.x += a.x; acc.y += a.y; acc.z += a.z; acc.w += a.w;
    }
    ((float4*)d.out)[o] = acc;
    if (d.stats) {
      const float a[4] = {acc.x, acc.y, acc.z, acc.w};
      if (fixed_c) {   // this thread always sees the same four channels: keep their sums in registers
#pragma unroll
        for (int j = 0; j < 4; ++j) { rs[j] += a[j]; rq[j] = fmaf(a[j], a[j], rq[j]); }
      } else {
        const int cpg = d.C / d.G;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int g = (c4 * 4 + j) / cpg;
          atomicAdd(&sstat[g], (double)a[j]);
          atomicAdd(&sstat[d.G + g], (double)(a[j] * a[j]));
        }
      }
    }
  }
  if (d.stats) {
    if (fixed_c && (long long)blockIdx.x * blockDim.x + threadIdx.x < per_n) {
      const int cpg = d.C / d.G;
      const int c4 = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) % c4n);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int g = (c4 * 4 + j) / cpg;
        atomicAdd(&sstat[g], (double)rs[j]);
        atomicAdd(&sstat[d.G + g], (double)rq[j]);
      }
    }
    __syncthreads();
    for (int g = threadIdx.x; g < d.G; g += blockDim.x) {
      atomicAdd(&d.stats[((long long)n * d.G + g) * 2], sstat[g]);
      atomicAdd(&d.stats[((long long)n * d.G + g) * 2 + 1], sstat[d.G + g]);
    }
  }
}

// avgpool with kernel == stride == (fd, fh, fw), channels-last; optional add + stats of the result
__global__ void __launch_bounds__(256) avgpool_kernel(const emo_resample_desc d) {
  const int c4n = d.C >> 2;
  const int Do = d.D / d.fd, Ho = d.H / d.fh, Wo = d.W / d.fw;
  const long long per_n = (long long)Do * Ho * Wo * c4n;
  const int n = blockIdx.y;
  extern __shared__ double sstat[];
  if (d.stats) {
    for (int i = threadIdx.x; i < 2 * d.G; i += blockDim.x) sstat[i] = 0.0;
    __syncthreads();
  }
  const float4* x4 = (const float4*)d.x + (long long)n * d.D * d.H * d.W * c4n;
  const float inv = 1.f / (float)(d.fd * d.fh * d.fw);
  const bool fixed_c = ((long long)gridDim.x * blockDim.x) % c4n == 0;  // see upsample_trilinear_kernel
  float rs[4] = {0.f, 0.f, 0.f, 0.f}, rq[4] = {0.f, 0.f, 0.f, 0.f};
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < per_n; t += (long long)gridDim.x * blockDim.x) {
    // 32-bit index arithmetic (the host requires per_n < 2^31): the 64-bit form is four emulated divisions per float4
    const unsigned tu = (unsigned)t;
    const int c4 = (int)(tu % (unsigned)c4n);
    unsigned s = tu / (unsigned)c4n;
    const int ow = (int)(s % (unsigned)Wo); s /= (unsigned)Wo;
    const int oh = (int)(s % (unsigned)Ho); s /= (unsigned)Ho;
    const int od = (int)s;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int a = 0; a < d.fd; ++a)
      for (int b = 0; b < d.fh; ++b)
        for (int c = 0; c < d.fw; ++c) {
          const float4 v = __ldg(x4 + (((long long)(od * d.fd + a) * d.H + (oh * d.fh + b)) * d.W + (ow * d.fw + c)) * c4n + c4);
          acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
    acc.x *= inv; acc.y *= inv; acc.z *= inv; acc.w *= inv;
    const long long o = (long long)n * per_n + t;
    if (d.add) {
      const float4 a = __ldg((const float4*)d.add + o);
      acc.x += a.x; acc.y += a.y; acc.z += a.z; acc.w += a.w;
    }
    ((float4*)d.out)[o] = acc;
    if (d.stats) {
      const float a[4] = {acc.x, acc.y, acc.z, acc.w};
      if (fixed_c) {   // this thread always sees the same four channels: keep their sums in registers
#pragma unroll
        for (int j = 0; j < 4; ++j) { rs[j] += a[j]; rq[j] = fmaf(a[j], a[j], rq[j]); }
      } else {
        const int cpg = d.C / d.G;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int g = (c4 * 4 + j) / cpg;
          atomicAdd(&sstat[g], (double)a[j]);
          atomicAdd(&sstat[d.G + g], (double)(a[j] * a[j]));
        }
      }
    }
  }
  if (d.stats) {
    if (fixed_c && (long long)blockIdx.x * blockDim.x + threadIdx.x < per_n) {
      const int cpg = d.C / d.G;
      const int c4 = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) % c4n);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int g = (c4 * 4 + j) / cpg;
        atomicAdd(&sstat[g], (double)rs[j]);
        atomicAdd(&sstat[d.G + g], (double)rq[j]);
      }
    }
    __syncthreads();
    for (int g = threadIdx.x; g < d.G; g += blockDim.x) {
      atomicAdd(&d.stats[((long long)n * d.G + g) * 2], sstat[g]);
      atomicAdd(&d.stats[((long long)n * d.G + g) * 2 + 1], sstat[d.G + g]);
    }
  }
}

__global__ void maxpool3x3s2_kernel(const float* __restrict__ x, int N, int H, int W, int C, float* __restrict__ out) {
  const int c4n = C >> 2;
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  const long long total = (long long)N * Ho * Wo * c4n;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(t % c4n);
    long long s = t / c4n;
    const int ow = (int)(s % Wo); s /= Wo;
    const int oh = (int)(s % Ho); s /= Ho;
    const int n = (int)s;
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = oh * 2 + ky - 1;
      if (iy < 0 || iy >= H) continue;
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = ow * 2 + kx - 1;
        if (ix < 0 || ix >= W) continue;
        const float4 v = __ldg((const float4*)x + (((long long)n * H + iy) * W + ix) * c4n + c4);
        m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
      }
    }
    ((float4*)out)[t] = m;
  }
}

__global__ void global_avgpool_kernel(const float* __restrict__ x, int N, long long S, int C, float* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * C) return;
  const int n = idx / C, c = idx % C;
  float acc = 0.f;
  for (long long s = 0; s < S; ++s) acc += x[((long long)n * S + s) * C + c];
  out[idx] = acc / (float)S;
}

// ------------------------------------------------------------------------------------------------
// pose algebra: pose_math.cuh (host+device source, also compiled for the CPU by tests/test_pose_math_host.py)
// ------------------------------------------------------------------------------------------------
__global__ void pose_theta_kernel(const emo_pose_desc d) {
  if (d.smooth_state) {
    // exponential smoothing carries state from sample to sample: one thread walks the samples in order
    if (blockIdx.x == 0 && threadIdx.x == 0)
      for (int n = 0; n < d.N; ++n) pose::pose_sample(d, n);
    return;
  }
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n < d.N) pose::pose_sample(d, n);
}

// video-loop compositing (E_emo_infer_video.ipynb cell 41): out = m^8 * img + (1 - m^8) * bg with m zeroed below the threshold
__global__ void __launch_bounds__(256) composite_kernel(const float* __restrict__ img, const float* __restrict__ mask, const float* __restrict__ bg,
                                                       int N, int C, long long HW, float thr, float* __restrict__ out) {
  const long long total = (long long)N * C * HW;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const long long s = t % HW;
    const long long nc = t / HW;
    const int c = (int)(nc % C);
    const long long n = nc / C;
    out[t] = composite_pixel(__ldg(mask + n * HW + s), img + t, bg + (long long)c * HW + s, thr);
  }
}

}  // namespace emo

using namespace emo;

extern "C" int emo_composite(const float* img, const float* mask, const float* bg, int N, int C, int H, int W, float threshold, float* out, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(img && mask && bg && out && N > 0 && C > 0 && H > 0 && W > 0, "emo_composite: bad arguments");
  const long long total = (long long)N * C * H * W;
  long long blocks = cdivll(total, 256);
  if (blocks > 132ll * 16) blocks = 132ll * 16;
  launch_kernel(composite_kernel, (unsigned)blocks, 256, 0, stream, img, mask, bg, N, C, (long long)H * W, threshold, out);
  return check_launch("emo_composite");
}

extern "C" const char* emo_last_error(void) { return emo::g_err; }
extern "C" int emo_version(void) { return 111; }  // 101: emo_pose_desc (+theta_in, mix_old, smoothing) and emo_conv_desc (+upconv) grew trailing fields

extern "C" int emo_device_info(int* sm_count, int* cc) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) { set_error("emo_device_info: %s", cudaGetErrorString(e)); return EMO_ERR_CUDA; }
  int sms = 0, major = 0, minor = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (sm_count) *sm_count = sms;
  if (cc) *cc = major * 10 + minor;
  return EMO_OK;
}

extern "C" int emo_linear(const emo_linear_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(d && d->x && d->w && d->out, "emo_linear: null pointer");
  EMO_REQUIRE(d->M > 0 && d->N > 0 && d->K > 0, "emo_linear: bad shape");
  const long long warps = (long long)d->M * d->N;
  launch_kernel(linear_kernel, (unsigned)cdivll(warps * 32, 256), 256, 0, stream, *d);
  return check_launch("emo_linear");
}

extern "C" int emo_conv_direct(const emo_conv_direct_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(d && d->x && d->w && d->out, "emo_conv_direct: null pointer");
  EMO_REQUIRE(d->Cout % 4 == 0, "emo_conv_direct: Cout must be a multiple of 4");
  const long long per_n = (long long)d->Hout * d->Wout * (d->Cout / 4);
  if (d->stats) EMO_REQUIRE(per_n % 256 == 0 && d->G > 0 && d->Cout % d->G == 0, "emo_conv_direct: stats need Hout*Wout*Cout/4 %% 256 == 0");
  const long long total = per_n * d->N;
  launch_kernel(conv_direct_kernel, (unsigned)cdivll(total, 256), 256, d->stats ? 2 * d->G * sizeof(double) : 0, stream, *d);
  return check_launch("emo_conv_direct");
}

extern "C" int emo_stem_pack(const float* x, int N, int H, int W, int C, float scale, void* out, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(x && out, "emo_stem_pack: null pointer");
  EMO_REQUIRE(((uintptr_t)x % 16) == 0 && ((uintptr_t)out % 16) == 0, "emo_stem_pack: x and out must be 16-byte aligned");
  EMO_REQUIRE(C == 4, "emo_stem_pack: C must be 4 (C=%d)", C);
  EMO_REQUIRE(N > 0 && H > 0 && W > 0, "emo_stem_pack: bad shape (N=%d H=%d W=%d)", N, H, W);
  EMO_REQUIRE(scale > 0.f, "emo_stem_pack: scale must be positive");
  const long long pixels = (long long)N * H * W;
  long long blocks = cdivll(pixels, 256);
  if (blocks > 132ll * 16) blocks = 132ll * 16;
  launch_kernel(stem_pack_kernel, (unsigned)blocks, 256, 0, stream, (const float4*)x, H, W, pixels, scale, (uint4*)out);
  return check_launch("emo_stem_pack");
}

static int resample_check(const emo_resample_desc* d, const char* who) {
  EMO_REQUIRE(d && d->x && d->out, "%s: null pointer", who);
  EMO_REQUIRE(d->C % 4 == 0, "%s: C must be a multiple of 4", who);
  EMO_REQUIRE((d->fd == 1 || d->fd == 2) && (d->fh == 1 || d->fh == 2) && (d->fw == 1 || d->fw == 2), "%s: factors must be 1 or 2", who);
  if (d->stats) EMO_REQUIRE(d->G > 0 && d->C % d->G == 0, "%s: C not divisible by G", who);
  return EMO_OK;
}

extern "C" int emo_upsample_trilinear(const emo_resample_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  int rc = resample_check(d, "emo_upsample_trilinear");
  if (rc) return rc;
  const long long per_n = (long long)d->D * d->fd * d->H * d->fh * d->W * d->fw * (d->C / 4);
  EMO_REQUIRE(per_n < (1ll << 31), "emo_upsample_trilinear: more than 2^31 output vectors per sample");
  long long bx = cdivll(per_n, 256 * 4);
  if (bx > 132 * 16) bx = 132 * 16;
  if (bx < 1) bx = 1;
  dim3 grid((unsigned)bx, (unsigned)d->N);
  launch_kernel(upsample_trilinear_kernel, grid, 256, d->stats ? 2 * d->G * sizeof(double) : 0, stream, *d);
  return check_launch("emo_upsample_trilinear");
}

extern "C" int emo_avgpool(const emo_resample_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  int rc = resample_check(d, "emo_avgpool");
  if (rc) return rc;
  EMO_REQUIRE(d->D % d->fd == 0 && d->H % d->fh == 0 && d->W % d->fw == 0, "emo_avgpool: size not divisible by the kernel");
  const long long per_n = (long long)(d->D / d->fd) * (d->H / d->fh) * (d->W / d->fw) * (d->C / 4);
  EMO_REQUIRE(per_n < (1ll << 31), "emo_avgpool: more than 2^31 output vectors per sample");
  long long bx = cdivll(per_n, 256 * 4);
  if (bx > 132 * 16) bx = 132 * 16;
  if (bx < 1) bx = 1;
  dim3 grid((unsigned)bx, (unsigned)d->N);
  launch_kernel(avgpool_kernel, grid, 256, d->stats ? 2 * d->G * sizeof(double) : 0, stream, *d);
  return check_launch("emo_avgpool");
}

extern "C" int emo_maxpool2d_3x3s2(const float* x, int N, int H, int W, int C, float* out, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(x && out && C % 4 == 0, "emo_maxpool2d_3x3s2: bad arguments");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const long long total = (long long)N * Ho * Wo * (C / 4);
  launch_kernel(maxpool3x3s2_kernel, (unsigned)cdivll(total, 256), 256, 0, stream, x, N, H, W, C, out);
  return check_launch("emo_maxpool2d_3x3s2");
}

extern "C" int emo_global_avgpool(const float* x, int N, long long S, int C, float* out, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(x && out, "emo_global_avgpool: null pointer");
  launch_kernel(global_avgpool_kernel, cdiv(N * C, 128), 128, 0, stream, x, N, S, C, out);
  return check_launch("emo_global_avgpool");
}

extern "C" int emo_pose_theta(const emo_pose_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(d && (d->srt || d->theta_in), "emo_pose_theta: srt or theta_in is required");
  EMO_REQUIRE(d->N > 0, "emo_pose_theta: N must be positive (N=%d)", d->N);
  EMO_REQUIRE(!d->mix || d->source_theta, "emo_pose_theta: mix needs source_theta");
  EMO_REQUIRE(!d->smooth_state || (d->smooth_momentum >= 0.f && d->smooth_momentum <= 1.f),
              "emo_pose_theta: smooth_momentum must be in [0,1]");
  EMO_REQUIRE(!d->smooth_state || (d->smooth_one_minus >= 0.f && d->smooth_one_minus <= 1.f),
              "emo_pose_theta: smooth_one_minus must be in [0,1]");
  // a value that does not belong to the momentum would smooth with the wrong weights; fp32(1 - m) and 1 - fp32(m) differ
  // by under 2^-23.  Zero stands for "derive it from smooth_momentum" (pose_math.cuh)
  EMO_REQUIRE(!d->smooth_state || d->smooth_one_minus == 0.f ||
                  fabs((double)d->smooth_one_minus - (1.0 - (double)d->smooth_momentum)) <= 0x1p-23,
              "emo_pose_theta: smooth_one_minus must be 1 - smooth_momentum (%.9g, %.9g)", d->smooth_one_minus,
              d->smooth_momentum);
  launch_kernel(pose_theta_kernel, cdiv(d->N, 32), 32, 0, stream, *d);
  return check_launch("emo_pose_theta");
}
