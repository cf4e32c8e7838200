// grid_sample kernels (HBM-bound; see DESIGN.md "grid_sample_3d").
//
//  emo_grid_sample3d        trilinear, zeros padding, align_corners=False
//     replaces models/stage_1/volumetric_avatar/va.py:261-265 (F.grid_sample on a 5-D volume) and, with
//     `theta`, also the affine lattice build notebooks/infer.py:441-444 / :583-588
//     (identity_grid_3d (va.py:101-105: linspace(-1,1,n) per axis, [x,y,z,1]) . theta[:, :3]^T), so the
//     (N,D,H,W,3) grid tensor never exists in HBM.
//  emo_grid_sample2d_affine bilinear face alignment of expression_embedder.py:224-231.
//  emo_resize_bilinear      F.interpolate(mode='bilinear') of head_pose_regressor.py:24-25.
//
// Un-normalisation (align_corners=False): ix = ((x + 1) * W - 1) / 2  (utils.py:24-27 restates it).
#include <stdlib.h>

#include "common.cuh"

namespace emo {

struct GS3Params {
  const float* in;
  const float* grid;
  const float* theta;
  int N, C, Din, Hin, Win, Dout, Hout, Wout;
  float* out;
  __nv_bfloat16* out_hi;
  __nv_bfloat16* out_lo;
  __nv_bfloat16* out_lo2;
  long long os_n, os_c, os_d, os_h, os_w;
  int plane_fp16;     // one fp16 plane of y * plane_scale in out_hi (out_lo / out_lo2 NULL)
  float plane_scale;
  // brick decomposition of the output lattice (channels-last kernel)
  int bw, bh, bd, bricks_w, bricks_h, bricks_d;
};

// linspace(-1, 1, n)[i] exactly as torch computes it (start + i*step for the first half,
// end - (n-1-i)*step for the second half; step = 2/(n-1) in fp32).
__device__ __forceinline__ float lin_m1_p1(int i, int n) {
  if (n == 1) return -1.f;
  const float step = 2.0f / (float)(n - 1);
  return (i < n / 2) ? (-1.f + step * (float)i) : (1.f - step * (float)(n - 1 - i));
}

__device__ __forceinline__ void sample_coord(const GS3Params& p, int n, int od, int oh, int ow, float& gx, float& gy, float& gz) {
  if (p.theta) {
    const float* t = p.theta + n * 12;
    const float u = lin_m1_p1(ow, p.Wout), v = lin_m1_p1(oh, p.Hout), w = lin_m1_p1(od, p.Dout);
    // bmm row . column in the order torch accumulates a 4-term dot: ((u*t0 + v*t1) + w*t2) + 1*t3
    gx = fmaf(w, t[2], fmaf(v, t[1], u * t[0])) + t[3];
    gy = fmaf(w, t[6], fmaf(v, t[5], u * t[4])) + t[7];
    gz = fmaf(w, t[10], fmaf(v, t[9], u * t[8])) + t[11];
  } else {
    const float* g = p.grid + ((((long long)n * p.Dout + od) * p.Hout + oh) * p.Wout + ow) * 3;
    gx = __ldg(g); gy = __ldg(g + 1); gz = __ldg(g + 2);
  }
}

// L2 eviction-priority hints: the volume is re-read by neighbouring voxels' corner fetches (evict_last), the output is
// written once and not read by this kernel (evict_first).  Measured with tools/gs3_lab (round 2, bit-identical output):
// 16 x 64 x 64 warp-field case 22.6 -> 20.6 us, 64^3 cases unchanged or 2% better.
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t l2_policy_evict_normal() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ float4 ldg_hint(const float4* p, uint64_t pol) {
  float4 v;
  asm volatile("ld.global.nc.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void stg_hint(float4* p, const float4& v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}

struct Corner8 {
  int x0, y0, z0;
  float fx, fy, fz;
};

__device__ __forceinline__ Corner8 corners(const GS3Params& p, float gx, float gy, float gz) {
  const float ix = ((gx + 1.f) * (float)p.Win - 1.f) * 0.5f;
  const float iy = ((gy + 1.f) * (float)p.Hin - 1.f) * 0.5f;
  const float iz = ((gz + 1.f) * (float)p.Din - 1.f) * 0.5f;
  const float x0 = floorf(ix), y0 = floorf(iy), z0 = floorf(iz);
  Corner8 c;
  // clamp before the int conversion so that wild coordinates stay out of range instead of overflowing
  c.x0 = (int)fminf(fmaxf(x0, -2.f), (float)p.Win + 1.f);
  c.y0 = (int)fminf(fmaxf(y0, -2.f), (float)p.Hin + 1.f);
  c.z0 = (int)fminf(fmaxf(z0, -2.f), (float)p.Din + 1.f);
  c.fx = ix - x0; c.fy = iy - y0; c.fz = iz - z0;
  return c;
}

// ------------------------------------------------------------------------------------------------
// channels-last kernel.  A CTA owns a compact (bd x bh x bw) brick of the output lattice (L1 reuse of the overlapping
// 8-corner footprints).  Phase 1: one thread per voxel computes the sample position, the eight clamped corner offsets
// and trilinear weights ONCE and parks them in shared memory (the per-voxel arithmetic is ~200 instructions; doing it
// in each of the C/4 channel threads made the kernel issue-bound).  Phase 2: one thread = one float4 of channels of
// one voxel: two 16-byte broadcast LDS pairs, eight 16-byte gathers issued back to back, 32 FMAs, one store.
// Every corner fetch is a 16-byte load inside a contiguous C*4-byte run.
// ------------------------------------------------------------------------------------------------
static constexpr int kBrickVox = 256;

template <bool SPLIT>
__global__ void __launch_bounds__(256) gs3_cl_kernel(const GS3Params p) {
  __shared__ __align__(16) int s_off[kBrickVox][8];
  __shared__ __align__(16) float s_wgt[kBrickVox][8];
  __shared__ long long s_out[kBrickVox];  // output element offset of the voxel (or -1)
  const int c4n = p.C >> 2;
  int b = blockIdx.x;
  const int bwi = b % p.bricks_w; b /= p.bricks_w;
  const int bhi = b % p.bricks_h; b /= p.bricks_h;
  const int bdi = b % p.bricks_d; b /= p.bricks_d;
  const int n = b;
  const int brick_vox = p.bw * p.bh * p.bd;  // <= kBrickVox
  {
    const int vox = threadIdx.x;
    if (vox < brick_vox) {
      const int lw = vox % p.bw, lh = (vox / p.bw) % p.bh, ld = vox / (p.bw * p.bh);
      const int ow = bwi * p.bw + lw, oh = bhi * p.bh + lh, od = bdi * p.bd + ld;
      long long o = -1;
      if (ow < p.Wout && oh < p.Hout && od < p.Dout) {
        float gx, gy, gz;
        sample_coord(p, n, od, oh, ow, gx, gy, gz);
        const Corner8 k = corners(p, gx, gy, gz);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int dx = j & 1, dy = (j >> 1) & 1, dz = j >> 2;
          const int x = k.x0 + dx, y = k.y0 + dy, z = k.z0 + dz;
          const bool ok = (unsigned)x < (unsigned)p.Win && (unsigned)y < (unsigned)p.Hin && (unsigned)z < (unsigned)p.Din;
          const int xc = min(max(x, 0), p.Win - 1), yc = min(max(y, 0), p.Hin - 1), zc = min(max(z, 0), p.Din - 1);
          s_wgt[vox][j] = ok ? (dx ? k.fx : 1.f - k.fx) * (dy ? k.fy : 1.f - k.fy) * (dz ? k.fz : 1.f - k.fz) : 0.f;
          s_off[vox][j] = ((zc * p.Hin + yc) * p.Win + xc) * c4n;
        }
        o = (long long)n * p.os_n + (long long)od * p.os_d + (long long)oh * p.os_h + (long long)ow * p.os_w;
      }
      s_out[vox] = o;
    }
  }
  __syncthreads();
  const int work = brick_vox * c4n;
  const float4* in4 = (const float4*)p.in + (long long)n * p.Din * p.Hin * p.Win * c4n;
  const uint64_t pol_in = l2_policy_evict_last(), pol_out = l2_policy_evict_first();
  for (int t = threadIdx.x; t < work; t += blockDim.x) {
    const int vox = t / c4n, c4 = t - vox * c4n;
    const long long ob = s_out[vox];
    if (ob < 0) continue;
    const int4 o0 = *(const int4*)&s_off[vox][0], o1 = *(const int4*)&s_off[vox][4];
    const float4 w0 = *(const float4*)&s_wgt[vox][0], w1 = *(const float4*)&s_wgt[vox][4];
    const float4* base = in4 + c4;
    const float4 v0 = ldg_hint(base + o0.x, pol_in), v1 = ldg_hint(base + o0.y, pol_in), v2 = ldg_hint(base + o0.z, pol_in), v3 = ldg_hint(base + o0.w, pol_in);
    const float4 v4 = ldg_hint(base + o1.x, pol_in), v5 = ldg_hint(base + o1.y, pol_in), v6 = ldg_hint(base + o1.z, pol_in), v7 = ldg_hint(base + o1.w, pol_in);
    float4 acc;
#define EMO_GS_ACC(f) \
  acc.f = fmaf(v7.f, w1.w, fmaf(v6.f, w1.z, fmaf(v5.f, w1.y, fmaf(v4.f, w1.x, \
          fmaf(v3.f, w0.w, fmaf(v2.f, w0.z, fmaf(v1.f, w0.y, v0.f * w0.x)))))));
    EMO_GS_ACC(x) EMO_GS_ACC(y) EMO_GS_ACC(z) EMO_GS_ACC(w)
#undef EMO_GS_ACC
    const long long o = ob + (long long)(c4 * 4) * p.os_c;
    if (p.os_c == 1) {
      if (p.out) stg_hint((float4*)(p.out + o), acc, pol_out);  // the output is not re-read by this kernel
      if (SPLIT) {
        uint2 hi, lo, lo2;
        if (p.plane_fp16) {
          *(uint2*)(p.out_hi + o) = plane4_h(acc, p.plane_scale);
        } else {
          if (p.out_lo2) {
            split4x3(acc, hi, lo, lo2);
            *(uint2*)(p.out_lo2 + o) = lo2;
          } else {
            split4(acc, hi, lo);
          }
          *(uint2*)(p.out_hi + o) = hi;
          *(uint2*)(p.out_lo + o) = lo;
        }
      }
    } else {
      const float a[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (p.out) p.out[o + j * p.os_c] = a[j];
        if (SPLIT && p.plane_fp16) {
          ((__half*)p.out_hi)[o + j * p.os_c] = f16_plane(a[j] * p.plane_scale);
        } else if (SPLIT) {
          __nv_bfloat16 h, l, l2;
          split_bf16x3(a[j], h, l, l2);
          if (!p.out_lo2) split_bf16(a[j], h, l);
          p.out_hi[o + j * p.os_c] = h;
          p.out_lo[o + j * p.os_c] = l;
          if (p.out_lo2) p.out_lo2[o + j * p.os_c] = l2;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Bulk-copy gather variant of the channels-last kernel ("TMA-staged feature tiles" in gather form; instrumented build only until
// measured: EMO_GS3_BULK=1, tools/gs3_check and tools/gs3_lab).  The eight corner rows of a voxel (C x 4 bytes each, contiguous in a
// channels-last volume) are fetched with cp.async.bulk (1-D bulk copies global -> shared memory, completion counted on an
// mbarrier) instead of LDG.128: the async proxy does not pay the L1tex wavefront cost that bounds the LSU path (~50 clk per voxel
// and SM at C = 96).  Warp 0 is the producer: lanes < BV set up one voxel each (sample position -> clamped corner offsets +
// trilinear weights -> shared memory; the grid coordinates of the NEXT stage are loaded before this stage's set-up), then all 32
// lanes issue the 8 x BV row copies.  The other threads are consumers, one float4 of one voxel each: wait for the stage, blend the
// eight rows from shared memory in the brick kernel's FMA order (bit-identical output), store.  NST stages ring; chunks of BV
// voxels go round-robin over the persistent CTAs in raster order, so the grid sweeps the lattice as one thin slab.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t gs_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void gs_mbar_init(uint64_t* b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(gs_smem_u32(b)), "r"(c)); }
__device__ __forceinline__ void gs_mbar_expect(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(gs_smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void gs_mbar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(gs_smem_u32(b)) : "memory"); }
__device__ __forceinline__ void gs_mbar_wait(uint64_t* b, uint32_t parity) {
  asm volatile("{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D_%=;\nbra W_%=;\nD_%=:\n}\n" ::"r"(gs_smem_u32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void gs_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(gs_smem_u32(dst)), "l"(src), "r"(bytes),
               "r"(gs_smem_u32(bar)) : "memory");
}

template <int BV, int NST, bool SPLIT>
__global__ void __launch_bounds__(1024, 1) gs3_bulk_kernel(const GS3Params p) {
  extern __shared__ __align__(128) uint8_t gs_sraw[];
  const int c4n = p.C >> 2;
  const uint32_t row_bytes = (uint32_t)p.C * 4u;
  float* ring = (float*)gs_sraw;  // [NST][BV][8][C]
  __shared__ __align__(16) float s_wgt[NST][BV][8];
  __shared__ long long s_out[NST][BV];
  __shared__ int s_row[BV * 8];
  __shared__ uint64_t full_bar[NST], empty_bar[NST];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ncw = (BV * c4n + 31) / 32;  // consumer warps (host launches exactly 1 + ncw warps)
  if (threadIdx.x == 0) {
    for (int i = 0; i < NST; ++i) { gs_mbar_init(&full_bar[i], 1); gs_mbar_init(&empty_bar[i], (uint32_t)ncw); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const long long per_sample = (long long)p.Dout * p.Hout * p.Wout;  // a multiple of BV (host): chunks never straddle samples
  const long long nchunks = per_sample * p.N / BV;
  const size_t stage_floats = (size_t)BV * 8 * p.C;
  if (warp == 0) {
    int it = 0;
    float gx = 0.f, gy = 0.f, gz = 0.f;
    auto coords = [&](long long ch) {
      if (lane < BV && ch < nchunks) {
        const long long v = ch * BV + lane;
        const int n = (int)(v / per_sample);
        long long r = v - (long long)n * per_sample;
        const int ow = (int)(r % p.Wout); r /= p.Wout;
        const int oh = (int)(r % p.Hout);
        const int od = (int)(r / p.Hout);
        sample_coord(p, n, od, oh, ow, gx, gy, gz);
      }
    };
    long long chunk = blockIdx.x;
    coords(chunk);
    for (; chunk < nchunks; chunk += gridDim.x, ++it) {
      const int slot = it % NST;
      const float cx = gx, cy = gy, cz = gz;
      coords(chunk + gridDim.x);
      if (it >= NST) gs_mbar_wait(&empty_bar[slot], (uint32_t)((it / NST) - 1) & 1u);
      const long long v0 = chunk * BV;
      const int n = (int)(v0 / per_sample);
      if (lane < BV) {
        long long r = v0 + lane - (long long)n * per_sample;
        const int ow = (int)(r % p.Wout); r /= p.Wout;
        const int oh = (int)(r % p.Hout);
        const int od = (int)(r / p.Hout);
        const Corner8 k = corners(p, cx, cy, cz);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int dx = j & 1, dy = (j >> 1) & 1, dz = j >> 2;
          const int x = k.x0 + dx, y = k.y0 + dy, z = k.z0 + dz;
          const bool ok = (unsigned)x < (unsigned)p.Win && (unsigned)y < (unsigned)p.Hin && (unsigned)z < (unsigned)p.Din;
          const int xc = min(max(x, 0), p.Win - 1), yc = min(max(y, 0), p.Hin - 1), zc = min(max(z, 0), p.Din - 1);
          s_wgt[slot][lane][j] = ok ? (dx ? k.fx : 1.f - k.fx) * (dy ? k.fy : 1.f - k.fy) * (dz ? k.fz : 1.f - k.fz) : 0.f;
          s_row[lane * 8 + j] = (zc * p.Hin + yc) * p.Win + xc;
        }
        s_out[slot][lane] = (long long)n * p.os_n + (long long)od * p.os_d + (long long)oh * p.os_h + (long long)ow * p.os_w;
      }
      __syncwarp();
      if (lane == 0) gs_mbar_expect(&full_bar[slot], (uint32_t)(BV * 8) * row_bytes);
      __syncwarp();
      const char* vol = (const char*)(p.in + (long long)n * p.Din * p.Hin * p.Win * p.C);
      float* dst = ring + (size_t)slot * stage_floats;
      for (int q = lane; q < BV * 8; q += 32) gs_bulk_g2s(dst + (size_t)q * p.C, vol + (long long)s_row[q] * row_bytes, row_bytes, &full_bar[slot]);
      __syncwarp();  // s_row is rewritten by the next stage
    }
  } else {
    const int t = (int)threadIdx.x - 32;
    const int vox = t / c4n, c4 = t - vox * c4n;
    const bool active = t < BV * c4n;
    const uint64_t pol_out = l2_policy_evict_first();
    int it = 0;
    for (long long chunk = blockIdx.x; chunk < nchunks; chunk += gridDim.x, ++it) {
      const int slot = it % NST;
      gs_mbar_wait(&full_bar[slot], (uint32_t)(it / NST) & 1u);
      if (active) {
        const float4 w0 = *(const float4*)&s_wgt[slot][vox][0], w1 = *(const float4*)&s_wgt[slot][vox][4];
        const float4* src = (const float4*)(ring + (size_t)slot * stage_floats + (size_t)vox * 8 * p.C) + c4;
        const float4 v0 = src[0 * c4n], v1 = src[1 * c4n], v2 = src[2 * c4n], v3 = src[3 * c4n];
        const float4 v4 = src[4 * c4n], v5 = src[5 * c4n], v6 = src[6 * c4n], v7 = src[7 * c4n];
        float4 acc;
#define EMO_GS_ACC(f) \
  acc.f = fmaf(v7.f, w1.w, fmaf(v6.f, w1.z, fmaf(v5.f, w1.y, fmaf(v4.f, w1.x, \
          fmaf(v3.f, w0.w, fmaf(v2.f, w0.z, fmaf(v1.f, w0.y, v0.f * w0.x)))))));
        EMO_GS_ACC(x) EMO_GS_ACC(y) EMO_GS_ACC(z) EMO_GS_ACC(w)
#undef EMO_GS_ACC
        const long long o = s_out[slot][vox] + (long long)(c4 * 4);
        if (p.out) stg_hint((float4*)(p.out + o), acc, pol_out);
        if (SPLIT) {
          uint2 hi, lo, lo2;
          if (p.plane_fp16) {
            *(uint2*)(p.out_hi + o) = plane4_h(acc, p.plane_scale);
          } else {
            if (p.out_lo2) {
              split4x3(acc, hi, lo, lo2);
              *(uint2*)(p.out_lo2 + o) = lo2;
            } else {
              split4(acc, hi, lo);
            }
            *(uint2*)(p.out_hi + o) = hi;
            *(uint2*)(p.out_lo + o) = lo;
          }
        }
      }
      __syncwarp();
      if (lane == 0) gs_mbar_arrive(&empty_bar[slot]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// NCDHW kernel (drop-in layout of F.grid_sample): one thread = one output voxel, loops over channels with the
// corner offsets/weights held in registers; lanes run along W so both the gathers and the stores coalesce.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gs3_nc_kernel(const GS3Params p) {
  const long long total = (long long)p.N * p.Dout * p.Hout * p.Wout;
  const long long plane_in = (long long)p.Din * p.Hin * p.Win;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    long long r = idx;
    const int ow = (int)(r % p.Wout); r /= p.Wout;
    const int oh = (int)(r % p.Hout); r /= p.Hout;
    const int od = (int)(r % p.Dout); r /= p.Dout;
    const int n = (int)r;
    float gx, gy, gz;
    sample_coord(p, n, od, oh, ow, gx, gy, gz);
    const Corner8 k = corners(p, gx, gy, gz);
    int off[8];
    float wgt[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int dx = j & 1, dy = (j >> 1) & 1, dz = j >> 2;
      const int x = k.x0 + dx, y = k.y0 + dy, z = k.z0 + dz;
      const bool ok = x >= 0 && x < p.Win && y >= 0 && y < p.Hin && z >= 0 && z < p.Din;
      off[j] = ok ? ((z * p.Hin + y) * p.Win + x) : 0;
      wgt[j] = ok ? (dx ? k.fx : 1.f - k.fx) * (dy ? k.fy : 1.f - k.fy) * (dz ? k.fz : 1.f - k.fz) : 0.f;
    }
    const float* src = p.in + (long long)n * p.C * plane_in;
    const long long o = (long long)n * p.os_n + (long long)od * p.os_d + (long long)oh * p.os_h + (long long)ow * p.os_w;
    for (int c = 0; c < p.C; ++c) {
      const float* s = src + (long long)c * plane_in;
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc = fmaf(__ldg(s + off[j]), wgt[j], acc);
      if (p.out) p.out[o + (long long)c * p.os_c] = acc;
      if (p.out_hi && p.plane_fp16) {
        ((__half*)p.out_hi)[o + (long long)c * p.os_c] = f16_plane(acc * p.plane_scale);
      } else if (p.out_hi) {
        __nv_bfloat16 h, l, l2;
        split_bf16x3(acc, h, l, l2);
        if (!p.out_lo2) split_bf16(acc, h, l);
        p.out_hi[o + (long long)c * p.os_c] = h;
        p.out_lo[o + (long long)c * p.os_c] = l;
        if (p.out_lo2) p.out_lo2[o + (long long)c * p.os_c] = l2;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// 2-D affine bilinear sampler, NCHW in -> channels-last (padded) out, optional normalisation
// ------------------------------------------------------------------------------------------------
struct GS2Params {
  const float* in;
  int N, C, Hin, Win, Hout, Wout, C_pad;
  const float* theta;
  const float* mean;
  const float* std;
  float* out;
  float* out_nchw;
};

__global__ void gs2_affine_kernel(const GS2Params p) {
  const long long total = (long long)p.N * p.Hout * p.Wout;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    long long r = idx;
    const int ow = (int)(r % p.Wout); r /= p.Wout;
    const int oh = (int)(r % p.Hout); r /= p.Hout;
    const int n = (int)r;
    const float* t = p.theta + n * 6;
    const float u = lin_m1_p1(ow, p.Wout), v = lin_m1_p1(oh, p.Hout);
    const float gx = fmaf(v, t[1], u * t[0]) + t[2];
    const float gy = fmaf(v, t[4], u * t[3]) + t[5];
    const float ix = ((gx + 1.f) * (float)p.Win - 1.f) * 0.5f;
    const float iy = ((gy + 1.f) * (float)p.Hin - 1.f) * 0.5f;
    const float fx0 = floorf(ix), fy0 = floorf(iy);
    const int x0 = (int)fminf(fmaxf(fx0, -2.f), (float)p.Win + 1.f);
    const int y0 = (int)fminf(fmaxf(fy0, -2.f), (float)p.Hin + 1.f);
    const float fx = ix - fx0, fy = iy - fy0;
    float w[4];
    int off[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int dx = j & 1, dy = j >> 1;
      const int x = x0 + dx, y = y0 + dy;
      const bool ok = x >= 0 && x < p.Win && y >= 0 && y < p.Hin;
      off[j] = ok ? y * p.Win + x : 0;
      w[j] = ok ? (dx ? fx : 1.f - fx) * (dy ? fy : 1.f - fy) : 0.f;
    }
    for (int c = 0; c < p.C_pad; ++c) {
      float acc = 0.f;
      if (c < p.C) {
        const float* s = p.in + ((long long)n * p.C + c) * p.Hin * p.Win;
#pragma unroll
        for (int j = 0; j < 4; ++j) acc = fmaf(__ldg(s + off[j]), w[j], acc);
        if (p.out_nchw) p.out_nchw[(((long long)n * p.C + c) * p.Hout + oh) * p.Wout + ow] = acc;
        if (p.mean) acc = (acc - __ldg(p.mean + c)) / __ldg(p.std + c);
      }
      p.out[idx * p.C_pad + c] = acc;
    }
  }
}

// F.interpolate bilinear, align_corners=False, no antialias: src = (dst + 0.5) * scale - 0.5 clamped at 0
struct ResizeParams {
  const float* in;
  int N, C, Hin, Win, Hout, Wout, C_pad;
  const float* mean;
  const float* std;
  float* out;
};

// A bilinear_pixel source that reads composite_pixel(matte, img, bg) (composite_kernel's output, never written to memory) in
// place of an image value: image n of img (N,C,H,W) and matte (N,1,H,W), over bg (C,H,W).  bilinear_pixel offsets it by the
// channel plane (the matte has one plane) and then by the pixel, as it offsets a plain NCHW pointer.
struct CompositeAt {
  const float *img, *matte, *bg;
  float thr;
  __device__ __forceinline__ CompositeAt operator+(int i) const { return CompositeAt{img + i, matte + i, bg + i, thr}; }
};
struct CompositeSrc {
  const float *img, *matte, *bg;
  float thr;
  __device__ __forceinline__ CompositeSrc(const float* img, const float* matte, const float* bg, float thr, int n, int C, long long HW)
      : img(img + (long long)n * C * HW), matte(matte + n * HW), bg(bg), thr(thr) {}
  __device__ __forceinline__ CompositeAt operator+(long long plane) const { return CompositeAt{img + plane, matte, bg + plane, thr}; }
};
// bilinear_pixel's taps read __ldg(plane + offset); this overload makes that the composited value
using ::__ldg;
__device__ __forceinline__ float __ldg(const CompositeAt& p) { return composite_pixel(__ldg(p.matte), p.img, p.bg, p.thr); }

// One output pixel (n, oh, ow) of the bilinear resize, sh = Hin / Hout, sw = Win / Wout: for every channel c < C_pad,
// emit(c, v) with v = post(c, interpolation of input channel c) for c < C and v = 0 above.  resize_bilinear_kernel,
// s2_prepare_kernel and s2_prepare_composite_kernel all call it, so the stage-2 input is the same bits as emo_resize_bilinear's
// of the same input values.
template <class Src, class Post, class Emit>
__device__ __forceinline__ void bilinear_pixel(Src in, int n, int C, int C_pad, int Hin, int Win, int oh, int ow, float sh,
                                               float sw, Post post, Emit emit) {
  float sy = fmaxf(((float)oh + 0.5f) * sh - 0.5f, 0.f);
  float sx = fmaxf(((float)ow + 0.5f) * sw - 0.5f, 0.f);
  const int y0 = (int)sy, x0 = (int)sx;
  const int y1 = y0 + (y0 < Hin - 1 ? 1 : 0), x1 = x0 + (x0 < Win - 1 ? 1 : 0);
  const float ly = sy - (float)y0, lx = sx - (float)x0;
  const float hy = 1.f - ly, hx = 1.f - lx;
  for (int c = 0; c < C_pad; ++c) {
    float acc = 0.f;
    if (c < C) {
      const auto s = in + ((long long)n * C + c) * Hin * Win;
      acc = hy * (hx * __ldg(s + y0 * Win + x0) + lx * __ldg(s + y0 * Win + x1)) +
            ly * (hx * __ldg(s + y1 * Win + x0) + lx * __ldg(s + y1 * Win + x1));
      acc = post(c, acc);
    }
    emit(c, acc);
  }
}

__global__ void resize_bilinear_kernel(const ResizeParams p) {
  const long long total = (long long)p.N * p.Hout * p.Wout;
  const float sh = (float)p.Hin / (float)p.Hout, sw = (float)p.Win / (float)p.Wout;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    long long r = idx;
    const int ow = (int)(r % p.Wout); r /= p.Wout;
    const int oh = (int)(r % p.Hout); r /= p.Hout;
    const int n = (int)r;
    bilinear_pixel(p.in, n, p.C, p.C_pad, p.Hin, p.Win, oh, ow, sh, sw,
                   [&](int c, float acc) {
                     if (p.mean) acc = (acc - __ldg(p.mean + c)) / __ldg(p.std + c);
                     return acc;
                   },
                   [&](int c, float acc) { p.out[idx * p.C_pad + c] = acc; });
  }
}

// ------------------------------------------------------------------------------------------------
// the stage-1 -> stage-2 handoff of a refined frame (emo_s2_prepare, emo_s2_prepare_composite, emo_s2_masked_stem,
// emo_s2_finish, emo_s2_finish_masked)
// ------------------------------------------------------------------------------------------------
// One CTA = kS2Tile consecutive output pixels of one row of one image.  Each pixel's value (R, G, B, 0) is computed once and
// written by `out` (the NCHW `resized` image of the prepare passes) and as the stem's operand: the channels-last pixel itself
// (kStemX4, emo_resize_bilinear's layout with C_pad 4), or the 7 horizontal taps of emo_stem_pack's plane (kStemPlane),
// packed by plane4_h from the tile's values and a 3-pixel halo on each side, staged in shared memory; or no operand
// (kStemNone).
constexpr int kS2Tile = 256;
enum { kStemNone = 0, kStemX4 = 1, kStemPlane = 2 };

// The tile [w0, w0 + kS2Tile) of output row oh of image n: out(ow, pixel(ow)) and the stem's operand of the pixels.
template <int STEM, class Pixel, class Out>
__device__ __forceinline__ void s2_tile(int n, int oh, int w0, int S, Pixel pixel, Out out, float4* __restrict__ x4, uint4* __restrict__ plane,
                                        float scale, float4* row) {
  const int ow = w0 + (int)threadIdx.x;
  const long long HW = (long long)S * S;
  const long long pix = (long long)n * HW + (long long)oh * S + ow;
  if (STEM == kStemPlane) {
    for (int i = threadIdx.x; i < kS2Tile + 6; i += kS2Tile) {
      const int x = w0 + i - 3;
      row[i] = (x >= 0 && x < S) ? pixel(x) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
    if (ow >= S) return;
    const float4 v = row[threadIdx.x + 3];
    out(ow, v);
    uint2 t[8];
#pragma unroll
    for (int kx = 0; kx < 7; ++kx) {
      const int ix = ow + kx - 3;
      t[kx] = (ix >= 0 && ix < S) ? plane4_h(row[threadIdx.x + kx], scale) : make_uint2(0u, 0u);
    }
    t[7] = make_uint2(0u, 0u);
    uint4* o = plane + pix * 4;
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = make_uint4(t[2 * j].x, t[2 * j].y, t[2 * j + 1].x, t[2 * j + 1].y);
  } else {
    if (ow >= S) return;
    const float4 v = pixel(ow);
    out(ow, v);
    if (STEM == kStemX4) x4[pix] = v;
  }
}

// The prepare passes: pixel(n, oh, ow) is the bilinear resize of image n of the stage-1 image (plain, or composited), written to
// the NCHW `resized` image (N,3,S,S) and as the stem's operand.
template <int STEM, class Pixel>
__device__ __forceinline__ void s2_prepare_tile(int S, Pixel pixel_of, float* __restrict__ resized, float4* __restrict__ x4,
                                                uint4* __restrict__ plane, float scale, float4* row) {
  const int tiles = (S + kS2Tile - 1) / kS2Tile;
  const int w0 = (int)(blockIdx.x % tiles) * kS2Tile;
  const int oh = (int)((blockIdx.x / tiles) % S);
  const int n = (int)(blockIdx.x / ((long long)tiles * S));
  const auto pixel = [&](int ow) { return pixel_of(n, oh, ow); };
  const long long HW = (long long)S * S;
  const auto out = [&](int ow, const float4& v) {
    resized[(n * 3 + 0) * HW + (long long)oh * S + ow] = v.x;
    resized[(n * 3 + 1) * HW + (long long)oh * S + ow] = v.y;
    resized[(n * 3 + 2) * HW + (long long)oh * S + ow] = v.z;
  };
  s2_tile<STEM>(n, oh, w0, S, pixel, out, x4, plane, scale, row);
}

template <bool FP16>
__global__ void __launch_bounds__(kS2Tile) s2_prepare_kernel(const float* __restrict__ img, int Hin, int Win, int S, float sh, float sw,
                                                              float* __restrict__ resized, float4* __restrict__ x4, uint4* __restrict__ plane,
                                                              float scale) {
  __shared__ float4 row[kS2Tile + 6];
  const auto pixel = [&](int n, int oh, int ow) {
    float v[4];
    bilinear_pixel(img, n, 3, 4, Hin, Win, oh, ow, sh, sw, [](int, float acc) { return acc; }, [&](int c, float acc) { v[c] = acc; });
    return make_float4(v[0], v[1], v[2], v[3]);
  };
  s2_prepare_tile<FP16 ? kStemPlane : kStemX4>(S, pixel, resized, x4, plane, scale, row);
}

// s2_prepare_kernel of the composited image: every bilinear tap reads composite_pixel(matte, img, bg) (composite_kernel's value)
// in place of the stage-1 pixel.  matte (N,1,Hin,Win), bg (3,Hin,Win).
template <int STEM>
__global__ void __launch_bounds__(kS2Tile) s2_prepare_composite_kernel(const float* __restrict__ img, const float* __restrict__ matte,
                                                                        const float* __restrict__ bg, float thr, int Hin, int Win, int S,
                                                                        float sh, float sw, float* __restrict__ resized,
                                                                        float4* __restrict__ x4, uint4* __restrict__ plane, float scale) {
  __shared__ float4 row[kS2Tile + 6];
  const auto pixel = [&](int n, int oh, int ow) {
    float v[4];
    bilinear_pixel(CompositeSrc(img, matte, bg, thr, n, 3, (long long)Hin * Win), 0, 3, 4, Hin, Win, oh, ow, sh, sw,
                   [](int, float acc) { return acc; }, [&](int c, float acc) { v[c] = acc; });
    return make_float4(v[0], v[1], v[2], v[3]);
  };
  s2_prepare_tile<STEM>(S, pixel, resized, x4, plane, scale, row);
}

// The stem's operand of resized * matte (torch's x4 * mask of Stage2Model.forward: (R m, G m, B m, 0 m), one fp32 product each).
// resized (N,3,S,S), matte (N,1,S,S).
template <int STEM>
__global__ void __launch_bounds__(kS2Tile) s2_masked_stem_kernel(const float* __restrict__ resized, const float* __restrict__ matte, int S,
                                                                  float4* __restrict__ x4, uint4* __restrict__ plane, float scale) {
  __shared__ float4 row[kS2Tile + 6];
  const int tiles = (S + kS2Tile - 1) / kS2Tile;
  const int w0 = (int)(blockIdx.x % tiles) * kS2Tile;
  const int oh = (int)((blockIdx.x / tiles) % S);
  const int n = (int)(blockIdx.x / ((long long)tiles * S));
  const long long HW = (long long)S * S;
  const auto pixel = [&](int ow) {
    const long long s = (long long)oh * S + ow;
    const float m = __ldg(matte + n * HW + s);
    return make_float4(__fmul_rn(__ldg(resized + (n * 3 + 0) * HW + s), m), __fmul_rn(__ldg(resized + (n * 3 + 1) * HW + s), m),
                       __fmul_rn(__ldg(resized + (n * 3 + 2) * HW + s), m), __fmul_rn(0.f, m));
  };
  s2_tile<STEM>(n, oh, w0, S, pixel, [](int, const float4&) {}, x4, plane, scale, row);
}

// ffhq = clamp(x, 0, 1) as torch's clamp_ computes it (a NaN stays NaN) into out[i], and its uint8 value as image_to_u8_kernel
// writes it (trunc(clamp(x, 0, 1) * 255), NaN -> 0) into u8[o]
__device__ __forceinline__ void s2_store(float x, long long i, long long o, float* __restrict__ out, unsigned char* __restrict__ u8) {
  const float y = x != x ? x : fminf(fmaxf(x, 0.f), 1.f);
  out[i] = y;
  const float v = fminf(fmaxf(y, 0.f), 1.f) * 255.f;
  u8[o] = (unsigned char)(int)v;
}

// ffhq = clamp(resized + add, 0, 1) (one fp32 add) and its uint8 frame: thread = one pixel of the 3-channel NCHW images.
__global__ void __launch_bounds__(256) s2_finish_kernel(const float* __restrict__ resized, const float* __restrict__ add, int N, long long HW,
                                                        float* __restrict__ out, unsigned char* __restrict__ u8) {
  const long long total = (long long)N * HW;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const long long n = t / HW, s = t - n * HW;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const long long i = (n * 3 + c) * HW + s;
      s2_store(__fadd_rn(__ldg(resized + i), __ldg(add + i)), i, t * 3 + c, out, u8);
    }
  }
}

// s2_finish_kernel with the residual mask of Stage2Model.forward: clamp(resized + add * (matte * face), 0, 1) as torch computes
// it (fm = matte * face, add * fm, resized + add: one rounding each), face (N,1,H,W) uint8 0 / 1 or null (fm = matte).
__global__ void __launch_bounds__(256) s2_finish_masked_kernel(const float* __restrict__ resized, const float* __restrict__ add,
                                                               const float* __restrict__ matte, const unsigned char* __restrict__ face, int N,
                                                               long long HW, float* __restrict__ out, unsigned char* __restrict__ u8) {
  const long long total = (long long)N * HW;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const long long n = t / HW, s = t - n * HW;
    const float m = __ldg(matte + t);
    const float fm = face ? __fmul_rn(m, (float)face[t]) : m;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const long long i = (n * 3 + c) * HW + s;
      s2_store(__fadd_rn(__ldg(resized + i), __fmul_rn(__ldg(add + i), fm)), i, t * 3 + c, out, u8);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// wrapper-boundary image conversions and the bicubic pre-processing resize
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) u8_to_image_kernel(const unsigned char* __restrict__ in, int N, long long HW, int C, float* __restrict__ out) {
  const long long total = (long long)N * HW;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const long long n = t / HW, s = t - n * HW;
    for (int c = 0; c < C; ++c) out[(n * C + c) * HW + s] = __fdiv_rn((float)in[t * C + c], 255.f);  // ToTensor: u / 255
  }
}

__global__ void __launch_bounds__(256) image_to_u8_kernel(const float* __restrict__ in, int N, int C, long long HW, unsigned char* __restrict__ out) {
  const long long total = (long long)N * HW;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const long long n = t / HW, s = t - n * HW;
    for (int c = 0; c < C; ++c) {
      const float v = fminf(fmaxf(__ldg(in + (n * C + c) * HW + s), 0.f), 1.f) * 255.f;  // clamp(0, 1).mul(255).byte(): truncation
      out[t * C + c] = (unsigned char)(int)v;
    }
  }
}

// torch's upsample_bicubic2d (align_corners = False): src = scale * (dst + 0.5) - 0.5 (not clamped), taps floor(src) - 1 ..
// + 2 with indices clamped to the border, cubic-convolution coefficients with A = -0.75 evaluated as torch evaluates them
__device__ __forceinline__ void cubic_coeffs(float t, float (&w)[4]) {
  const float A = -0.75f;
  const float x0 = t + 1.f, x1 = t, x2 = 1.f - t, x3 = 2.f - t;
  w[0] = ((A * x0 - 5.f * A) * x0 + 8.f * A) * x0 - 4.f * A;
  w[1] = ((A + 2.f) * x1 - (A + 3.f)) * x1 * x1 + 1.f;
  w[2] = ((A + 2.f) * x2 - (A + 3.f)) * x2 * x2 + 1.f;
  w[3] = ((A * x3 - 5.f * A) * x3 + 8.f * A) * x3 - 4.f * A;
}

__global__ void __launch_bounds__(256) resize_bicubic_kernel(const float* __restrict__ in, int NC, int Hin, int Win, int Hout, int Wout,
                                                             float* __restrict__ out) {
  const float sh = (float)Hin / (float)Hout, sw = (float)Win / (float)Wout;
  const long long total = (long long)NC * Hout * Wout;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int ow = (int)(t % Wout);
    const int oh = (int)((t / Wout) % Hout);
    const long long nc = t / ((long long)Wout * Hout);
    const float ry = sh * ((float)oh + 0.5f) - 0.5f, rx = sw * ((float)ow + 0.5f) - 0.5f;
    const float fy = floorf(ry), fx = floorf(rx);
    float wy[4], wx[4];
    cubic_coeffs(ry - fy, wy);
    cubic_coeffs(rx - fx, wx);
    const float* src = in + nc * (long long)Hin * Win;
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int y = min(max((int)fy - 1 + i, 0), Hin - 1);
      float row = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int x = min(max((int)fx - 1 + j, 0), Win - 1);
        row += __ldg(src + (long long)y * Win + x) * wx[j];
      }
      acc += row * wy[i];
    }
    out[t] = acc;
  }
}

}  // namespace emo

using namespace emo;

extern "C" int emo_u8_to_image(const unsigned char* nhwc, int N, int H, int W, int C, float* nchw, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(nhwc && nchw && N > 0 && H > 0 && W > 0 && C > 0 && C <= 4, "emo_u8_to_image: bad arguments");
  const long long total = (long long)N * H * W;
  long long blocks = cdivll(total, 256);
  if (blocks > 132ll * 16) blocks = 132ll * 16;
  launch_kernel(u8_to_image_kernel, (unsigned)blocks, 256, 0, stream, nhwc, N, (long long)H * W, C, nchw);
  return check_launch("emo_u8_to_image");
}

extern "C" int emo_image_to_u8(const float* nchw, int N, int C, int H, int W, unsigned char* nhwc, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(nhwc && nchw && N > 0 && H > 0 && W > 0 && C > 0 && C <= 4, "emo_image_to_u8: bad arguments");
  const long long total = (long long)N * H * W;
  long long blocks = cdivll(total, 256);
  if (blocks > 132ll * 16) blocks = 132ll * 16;
  launch_kernel(image_to_u8_kernel, (unsigned)blocks, 256, 0, stream, nchw, N, C, (long long)H * W, nhwc);
  return check_launch("emo_image_to_u8");
}

extern "C" int emo_resize_bicubic(const float* in, int N, int C, int Hin, int Win, int Hout, int Wout, float* out, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(in && out && N > 0 && C > 0 && Hin > 0 && Win > 0 && Hout > 0 && Wout > 0, "emo_resize_bicubic: bad arguments");
  const long long total = (long long)N * C * Hout * Wout;
  long long blocks = cdivll(total, 256);
  if (blocks > 132ll * 16) blocks = 132ll * 16;
  launch_kernel(resize_bicubic_kernel, (unsigned)blocks, 256, 0, stream, in, N * C, Hin, Win, Hout, Wout, out);
  return check_launch("emo_resize_bicubic");
}

extern "C" int emo_grid_sample3d(const emo_grid_sample3d_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(d && d->in, "emo_grid_sample3d: null input");
  EMO_REQUIRE((d->grid != nullptr) != (d->theta != nullptr), "emo_grid_sample3d: exactly one of grid/theta must be given");
  EMO_REQUIRE(d->out || (d->out_hi && (d->out_lo || d->plane_fp16)), "emo_grid_sample3d: no output");
  EMO_REQUIRE((!d->out_lo || d->out_hi) && (!d->out_hi || d->out_lo || d->plane_fp16) && (!d->out_lo2 || d->out_lo),
              "emo_grid_sample3d: operand planes are out_hi + out_lo [+ out_lo2], or out_hi alone with plane_fp16");
  if (d->out_hi && d->plane_fp16)
    EMO_REQUIRE(!d->out_lo && !d->out_lo2 && d->plane_scale > 0.f,
                "emo_grid_sample3d: plane_fp16 writes one plane (out_lo, out_lo2 NULL) and needs plane_scale > 0");
  EMO_REQUIRE(d->N > 0 && d->C > 0 && d->Din > 0 && d->Hin > 0 && d->Win > 0 && d->Dout > 0 && d->Hout > 0 && d->Wout > 0,
              "emo_grid_sample3d: bad shape");
  GS3Params p;
  p.in = d->in; p.grid = d->grid; p.theta = d->theta;
  p.N = d->N; p.C = d->C; p.Din = d->Din; p.Hin = d->Hin; p.Win = d->Win;
  p.Dout = d->Dout; p.Hout = d->Hout; p.Wout = d->Wout;
  p.out = d->out; p.out_hi = (__nv_bfloat16*)d->out_hi; p.out_lo = (__nv_bfloat16*)d->out_lo;
  p.out_lo2 = (__nv_bfloat16*)d->out_lo2;
  p.os_n = d->os_n; p.os_c = d->os_c; p.os_d = d->os_d; p.os_h = d->os_h; p.os_w = d->os_w;
  p.plane_fp16 = d->out_hi ? d->plane_fp16 : 0; p.plane_scale = d->plane_scale;
  if (d->in_layout == 1) {
    EMO_REQUIRE(d->C % 4 == 0, "emo_grid_sample3d: channels-last path needs C %% 4 == 0 (C=%d)", d->C);
    EMO_REQUIRE(((uintptr_t)d->in % 16) == 0, "emo_grid_sample3d: input must be 16-byte aligned");
    if (d->os_c == 1)
      EMO_REQUIRE(d->os_n % 4 == 0 && d->os_d % 4 == 0 && d->os_h % 4 == 0 && d->os_w % 4 == 0,
                  "emo_grid_sample3d: vectorised output needs strides that are multiples of 4");
    EMO_REQUIRE((long long)d->Din * d->Hin * d->Win * (d->C / 4) < (1ll << 31), "emo_grid_sample3d: volume too large for 32-bit offsets");
    // SMs x resident CTAs (40 registers, 18 KB of shared memory -> 6 CTAs of 256 threads per SM), per device ordinal
    static int slots_dev[64][2] = {{0, 0}};
    static int sms_dev[64] = {0};
    const int k = d->out_hi ? 1 : 0;
    int dev = 0;
    {
      cudaError_t e0 = cudaGetDevice(&dev);
      EMO_REQUIRE(e0 == cudaSuccess, "emo_grid_sample3d: cudaGetDevice failed (%s)", cudaGetErrorString(e0));
    }
    int* slots = slots_dev[dev & 63];
    if (!slots[k]) {
      int sms = 0, occ = 0;
      cudaError_t e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
      if (e == cudaSuccess)
        e = k ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gs3_cl_kernel<true>, 256, 0)
              : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gs3_cl_kernel<false>, 256, 0);
      EMO_REQUIRE(e == cudaSuccess && sms > 0 && occ > 0, "emo_grid_sample3d: occupancy query failed (%s)", cudaGetErrorString(e));
      slots[k] = sms * occ;
      sms_dev[dev & 63] = sms;
    }
    // Brick shape = processing ORDER (tools/gs3_lab compares the shapes; every shape gives bit-identical output).  CTAs are
    // dispatched in blockIdx order (w fastest, then h, d, n), so the resident CTAs form a slab that sweeps through the lattice
    // along d.  With bricks of 8 x 8 x 4 = 256 voxels a 64^3 lattice is 1024 CTAs, about as many as are resident: the whole
    // lattice is in flight at once, and a warp-field tensor whose samples scatter over +-10 slices re-reads the 100 MB volume
    // from DRAM because the lines do not survive in L2 between their ~8 uses.  Small bricks keep the in-flight slab thin
    // (64-voxel bricks: 4096 CTAs, ~14 slices in flight).  A persistent kernel walking the same order with a barrier per chunk
    // is slower than letting the hardware dispatch small CTAs (tools/gs3_lab.cu keeps it).
    //   8 x 8 x 2 bricks (128 voxels) when that gives >= 4 waves of CTAs (batches), else compact 4 x 4 x 4 bricks (64 voxels:
    //   4096 CTAs for 64^3), 8 x 8 x 1 when the lattice is shallower than 4; small lattices then halve the brick height until
    //   there are >= 4 CTAs per SM.
    p.bw = d->Wout >= 8 ? 8 : d->Wout;
    p.bh = d->Hout >= 8 ? 8 : d->Hout;
    p.bd = d->Dout >= 2 ? 2 : d->Dout;
    if ((long long)d->N * cdiv(d->Wout, p.bw) * cdiv(d->Hout, p.bh) * cdiv(d->Dout, p.bd) < 4ll * slots[k]) {
      if (d->Dout >= 4 && d->Hout >= 4 && d->Wout >= 4) { p.bw = 4; p.bh = 4; p.bd = 4; }
      else p.bd = 1;
    }
    while ((long long)d->N * cdiv(d->Wout, p.bw) * cdiv(d->Hout, p.bh) * cdiv(d->Dout, p.bd) < 4ll * sms_dev[dev & 63] && p.bh > 2) p.bh >>= 1;
    unsigned threads = 256;
#ifdef EMO_CONV_DEBUG
    {  // instrumented build (tools/gs3_check): EMO_GS3_BRICK="bw,bh,bd[,threads]" forces the brick shape, read per call
      const char* bs = getenv("EMO_GS3_BRICK");
      int fw = 0, fh = 0, fd = 0, ft = 0;
      if (bs && sscanf(bs, "%d,%d,%d,%d", &fw, &fh, &fd, &ft) >= 3 && fw > 0 && fh > 0 && fd > 0 && fw * fh * fd <= kBrickVox) {
        p.bw = fw < d->Wout ? fw : d->Wout; p.bh = fh < d->Hout ? fh : d->Hout; p.bd = fd < d->Dout ? fd : d->Dout;
        if (ft >= p.bw * p.bh * p.bd && ft <= 256 && ft % 32 == 0) threads = (unsigned)ft;
      }
    }
#endif
#ifdef EMO_CONV_DEBUG
    {  // EMO_GS3_BULK=1: the bulk-copy gather variant where its preconditions hold (vector stores, whole stages, rows >= 256 B)
      const char* bk = getenv("EMO_GS3_BULK");
      constexpr int BV = 8, NST = 4;
      const long long per_sample = (long long)d->Dout * d->Hout * d->Wout;
      if (bk && atoi(bk) > 0 && d->os_c == 1 && per_sample % BV == 0 && d->C >= 64 && BV * (d->C / 4) <= 992) {
        const size_t smem = (size_t)NST * BV * 8 * d->C * 4;
        const int threads = 32 + cdiv(BV * (d->C / 4), 32) * 32;
        cudaError_t e = d->out_hi ? cudaFuncSetAttribute(gs3_bulk_kernel<BV, NST, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                                  : cudaFuncSetAttribute(gs3_bulk_kernel<BV, NST, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        int occ = 0;
        if (e == cudaSuccess)
          e = d->out_hi ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gs3_bulk_kernel<BV, NST, true>, threads, smem)
                        : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gs3_bulk_kernel<BV, NST, false>, threads, smem);
        EMO_REQUIRE(e == cudaSuccess && occ > 0, "emo_grid_sample3d: bulk variant does not fit (%s)", cudaGetErrorString(e));
        long long ctas = (long long)sms_dev[dev & 63] * occ;
        if (ctas > per_sample * d->N / BV) ctas = per_sample * d->N / BV;
        if (d->out_hi) launch_kernel(gs3_bulk_kernel<BV, NST, true>, (unsigned)ctas, (unsigned)threads, smem, stream, p);
        else launch_kernel(gs3_bulk_kernel<BV, NST, false>, (unsigned)ctas, (unsigned)threads, smem, stream, p);
        return check_launch("emo_grid_sample3d");
      }
    }
#endif
    p.bricks_w = cdiv(d->Wout, p.bw); p.bricks_h = cdiv(d->Hout, p.bh); p.bricks_d = cdiv(d->Dout, p.bd);
    const long long blocks = (long long)d->N * p.bricks_w * p.bricks_h * p.bricks_d;
    EMO_REQUIRE(blocks < (1ll << 31), "emo_grid_sample3d: grid too large");
    if (d->out_hi) launch_kernel(gs3_cl_kernel<true>, (unsigned)blocks, threads, 0, stream, p);
    else launch_kernel(gs3_cl_kernel<false>, (unsigned)blocks, threads, 0, stream, p);
  } else {
    p.bw = p.bh = p.bd = p.bricks_w = p.bricks_h = p.bricks_d = 1;
    const long long total = (long long)d->N * d->Dout * d->Hout * d->Wout;
    long long blocks = cdivll(total, 256);
    if (blocks > 132ll * 64) blocks = 132ll * 64;
    launch_kernel(gs3_nc_kernel, (unsigned)blocks, 256, 0, stream, p);
  }
  return check_launch("emo_grid_sample3d");
}

extern "C" int emo_grid_sample2d_affine(const emo_grid_sample2d_affine_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(d && d->in && d->theta && d->out, "emo_grid_sample2d_affine: null pointer");
  EMO_REQUIRE(d->C_pad >= d->C, "emo_grid_sample2d_affine: C_pad < C");
  GS2Params p{d->in, d->N, d->C, d->Hin, d->Win, d->Hout, d->Wout, d->C_pad, d->theta, d->mean, d->std, d->out, d->out_nchw};
  const long long total = (long long)d->N * d->Hout * d->Wout;
  launch_kernel(gs2_affine_kernel, (unsigned)cdivll(total, 128), 128, 0, stream, p);
  return check_launch("emo_grid_sample2d_affine");
}

extern "C" int emo_resize_bilinear(const emo_resize_bilinear_desc* d, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(d && d->in && d->out, "emo_resize_bilinear: null pointer");
  EMO_REQUIRE(d->C_pad >= d->C, "emo_resize_bilinear: C_pad < C");
  ResizeParams p{d->in, d->N, d->C, d->Hin, d->Win, d->Hout, d->Wout, d->C_pad, d->mean, d->std, d->out};
  const long long total = (long long)d->N * d->Hout * d->Wout;
  launch_kernel(resize_bilinear_kernel, (unsigned)cdivll(total, 128), 128, 0, stream, p);
  return check_launch("emo_resize_bilinear");
}

extern "C" int emo_s2_prepare(const float* img, int N, int Hin, int Win, int S, float* resized, float* x4, void* plane, float plane_scale,
                              void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(img && resized, "emo_s2_prepare: null pointer");
  EMO_REQUIRE((x4 != nullptr) != (plane != nullptr), "emo_s2_prepare: exactly one stem operand (x4 or plane) must be given");
  EMO_REQUIRE(N > 0 && Hin > 0 && Win > 0 && S > 0, "emo_s2_prepare: bad shape (N=%d Hin=%d Win=%d S=%d)", N, Hin, Win, S);
  EMO_REQUIRE(((uintptr_t)(x4 ? (const void*)x4 : plane) % 16) == 0, "emo_s2_prepare: the stem operand must be 16-byte aligned");
  if (plane) EMO_REQUIRE(plane_scale > 0.f, "emo_s2_prepare: plane_scale must be positive");
  const long long blocks = (long long)N * S * cdiv(S, kS2Tile);
  EMO_REQUIRE(blocks < (1ll << 31), "emo_s2_prepare: grid too large");
  const float sh = (float)Hin / (float)S, sw = (float)Win / (float)S;
  if (plane)
    launch_kernel(s2_prepare_kernel<true>, (unsigned)blocks, kS2Tile, 0, stream, img, Hin, Win, S, sh, sw, resized, (float4*)nullptr,
                  (uint4*)plane, plane_scale);
  else
    launch_kernel(s2_prepare_kernel<false>, (unsigned)blocks, kS2Tile, 0, stream, img, Hin, Win, S, sh, sw, resized, (float4*)x4,
                  (uint4*)nullptr, 0.f);
  return check_launch("emo_s2_prepare");
}

extern "C" int emo_s2_finish(const float* resized, const float* add, int N, int H, int W, float* out, unsigned char* u8, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(resized && add && out && u8, "emo_s2_finish: null pointer");
  EMO_REQUIRE(N > 0 && H > 0 && W > 0, "emo_s2_finish: bad shape (N=%d H=%d W=%d)", N, H, W);
  const long long total = (long long)N * H * W;
  long long blocks = cdivll(total, 256);
  if (blocks > 132ll * 16) blocks = 132ll * 16;
  launch_kernel(s2_finish_kernel, (unsigned)blocks, 256, 0, stream, resized, add, N, (long long)H * W, out, u8);
  return check_launch("emo_s2_finish");
}

static bool f32_aligned(const void* p) { return ((uintptr_t)p % 4) == 0; }

extern "C" int emo_s2_prepare_composite(const float* img, const float* matte, const float* bg, float threshold, int N, int Hin, int Win,
                                        int S, float* resized, float* x4, void* plane, float plane_scale, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(img && matte && bg && resized, "emo_s2_prepare_composite: null pointer");
  EMO_REQUIRE(!(x4 && plane), "emo_s2_prepare_composite: at most one stem operand (x4 or plane) may be given");
  EMO_REQUIRE(N > 0 && Hin > 0 && Win > 0 && S > 0, "emo_s2_prepare_composite: bad shape (N=%d Hin=%d Win=%d S=%d)", N, Hin, Win, S);
  EMO_REQUIRE(f32_aligned(img) && f32_aligned(matte) && f32_aligned(bg) && f32_aligned(resized),
              "emo_s2_prepare_composite: fp32 tensors must be 4-byte aligned");
  if (x4 || plane)
    EMO_REQUIRE(((uintptr_t)(x4 ? (const void*)x4 : plane) % 16) == 0, "emo_s2_prepare_composite: the stem operand must be 16-byte aligned");
  if (plane) EMO_REQUIRE(plane_scale > 0.f, "emo_s2_prepare_composite: plane_scale must be positive");
  const long long blocks = (long long)N * S * cdiv(S, kS2Tile);
  EMO_REQUIRE(blocks < (1ll << 31), "emo_s2_prepare_composite: grid too large");
  const float sh = (float)Hin / (float)S, sw = (float)Win / (float)S;
  const auto go = [&](auto kernel) {
    launch_kernel(kernel, (unsigned)blocks, kS2Tile, 0, stream, img, matte, bg, threshold, Hin, Win, S, sh, sw, resized, (float4*)x4,
                  (uint4*)plane, plane ? plane_scale : 0.f);
  };
  if (plane) go(s2_prepare_composite_kernel<kStemPlane>);
  else if (x4) go(s2_prepare_composite_kernel<kStemX4>);
  else go(s2_prepare_composite_kernel<kStemNone>);
  return check_launch("emo_s2_prepare_composite");
}

extern "C" int emo_s2_masked_stem(const float* resized, const float* matte, int N, int S, float* x4, void* plane, float plane_scale,
                                  void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(resized && matte, "emo_s2_masked_stem: null pointer");
  EMO_REQUIRE((x4 != nullptr) != (plane != nullptr), "emo_s2_masked_stem: exactly one stem operand (x4 or plane) must be given");
  EMO_REQUIRE(N > 0 && S > 0, "emo_s2_masked_stem: bad shape (N=%d S=%d)", N, S);
  EMO_REQUIRE(f32_aligned(resized) && f32_aligned(matte), "emo_s2_masked_stem: fp32 tensors must be 4-byte aligned");
  EMO_REQUIRE(((uintptr_t)(x4 ? (const void*)x4 : plane) % 16) == 0, "emo_s2_masked_stem: the stem operand must be 16-byte aligned");
  if (plane) EMO_REQUIRE(plane_scale > 0.f, "emo_s2_masked_stem: plane_scale must be positive");
  const long long blocks = (long long)N * S * cdiv(S, kS2Tile);
  EMO_REQUIRE(blocks < (1ll << 31), "emo_s2_masked_stem: grid too large");
  if (plane)
    launch_kernel(s2_masked_stem_kernel<kStemPlane>, (unsigned)blocks, kS2Tile, 0, stream, resized, matte, S, (float4*)nullptr,
                  (uint4*)plane, plane_scale);
  else
    launch_kernel(s2_masked_stem_kernel<kStemX4>, (unsigned)blocks, kS2Tile, 0, stream, resized, matte, S, (float4*)x4, (uint4*)nullptr,
                  0.f);
  return check_launch("emo_s2_masked_stem");
}

extern "C" int emo_s2_finish_masked(const float* resized, const float* add, const float* matte, const unsigned char* face, int N, int H,
                                    int W, float* out, unsigned char* u8, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(resized && add && matte && out && u8, "emo_s2_finish_masked: null pointer");
  EMO_REQUIRE(N > 0 && H > 0 && W > 0, "emo_s2_finish_masked: bad shape (N=%d H=%d W=%d)", N, H, W);
  EMO_REQUIRE(f32_aligned(resized) && f32_aligned(add) && f32_aligned(matte) && f32_aligned(out),
              "emo_s2_finish_masked: fp32 tensors must be 4-byte aligned");
  const long long total = (long long)N * H * W;
  long long blocks = cdivll(total, 256);
  if (blocks > 132ll * 16) blocks = 132ll * 16;
  launch_kernel(s2_finish_masked_kernel, (unsigned)blocks, 256, 0, stream, resized, add, matte, face, N, (long long)H * W, out, u8);
  return check_launch("emo_s2_finish_masked");
}
