// Shared device/host helpers for the emoportraits_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/emoportraits_b200.h"

namespace emo {

// ------------------------------------------------------------------------------------------------
// error plumbing (thread-local last-error string, see emo_last_error in the C-ABI)
// ------------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int check_launch(const char* what);

#define EMO_REQUIRE(cond, ...)                 \
  do {                                         \
    if (!(cond)) {                             \
      ::emo::set_error(__VA_ARGS__);           \
      return EMO_ERR_INVALID;                  \
    }                                          \
  } while (0)

// One launch path for every kernel of the library (cudaLaunchKernelEx).  Programmatic dependent launch (attribute +
// griddepcontrol.launch_dependents / .wait in every kernel) was built and measured in round 2: 221.8 vs 221.1 frames/s with one
// frame in flight, 254 vs 260 with two, 269 vs 270 with three (profiles/README.md) - the captured frame is a chain of
// data-dependent kernels whose summed durations already equal the frame time, so there is no launch gap to hide; removed.
#ifdef __CUDACC__
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#endif

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }
static inline long long cdivll(long long a, long long b) { return (a + b - 1) / b; }

// ------------------------------------------------------------------------------------------------
// fp32 -> (bf16 hi, bf16 lo) split.  x ~= hi + lo with |x - hi - lo| <= 2^-17 |x|.
// The three-product expansion hi*hi' + hi*lo' + lo*hi' then carries ~16 mantissa bits.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

__device__ __forceinline__ uint32_t pack_bf16x2(__nv_bfloat16 a, __nv_bfloat16 b) {
  return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}

// split 4 floats -> 2x uint2 (4 bf16 hi, 4 bf16 lo)
__device__ __forceinline__ void split4(const float4& v, uint2& hi, uint2& lo) {
  __nv_bfloat16 h0, h1, h2, h3, l0, l1, l2, l3;
  split_bf16(v.x, h0, l0);
  split_bf16(v.y, h1, l1);
  split_bf16(v.z, h2, l2);
  split_bf16(v.w, h3, l3);
  hi.x = pack_bf16x2(h0, h1);
  hi.y = pack_bf16x2(h2, h3);
  lo.x = pack_bf16x2(l0, l1);
  lo.y = pack_bf16x2(l2, l3);
}

// three-plane split: x ~= hi + lo + lo2 to ~2^-26 |x| (each residual is exact in fp32)
__device__ __forceinline__ void split_bf16x3(float x, __nv_bfloat16& hi, __nv_bfloat16& lo, __nv_bfloat16& lo2) {
  hi = __float2bfloat16_rn(x);
  const float r1 = x - __bfloat162float(hi);
  lo = __float2bfloat16_rn(r1);
  lo2 = __float2bfloat16_rn(r1 - __bfloat162float(lo));
}

__device__ __forceinline__ void split4x3(const float4& v, uint2& hi, uint2& lo, uint2& lo2) {
  __nv_bfloat16 h[4], l[4], m[4];
  split_bf16x3(v.x, h[0], l[0], m[0]);
  split_bf16x3(v.y, h[1], l[1], m[1]);
  split_bf16x3(v.z, h[2], l[2], m[2]);
  split_bf16x3(v.w, h[3], l[3], m[3]);
  hi.x = pack_bf16x2(h[0], h[1]); hi.y = pack_bf16x2(h[2], h[3]);
  lo.x = pack_bf16x2(l[0], l[1]); lo.y = pack_bf16x2(l[2], l[3]);
  lo2.x = pack_bf16x2(m[0], m[1]); lo2.y = pack_bf16x2(m[2], m[3]);
}

// ------------------------------------------------------------------------------------------------
// fp32 -> (fp16 hi, fp16 lo) split of a value pre-multiplied by a power of two: x*s ~= hi + lo to ~2^-22 |x*s| while the
// planes stay in fp16's normal range (|x*s| >= 2^-3 keeps lo normal; smaller values lose only absolute 2^-25).  Three
// fp16 MMAs (hi*hi + hi*lo + lo*hi) then carry ~22 mantissa bits: the fp32-faithful operand mode at half the MMAs of the
// three-plane bf16 mode (tools/split_precision_emulation.py: 7e-8 relative vs 6e-9 for bf16 x3 and 4e-6 for bf16 x2).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_f16x2(__half a, __half b) {
  return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}
__device__ __forceinline__ void split_f16(float x, __half& hi, __half& lo) {
  x = fminf(fmaxf(x, -65000.f), 65000.f);  // fp16 has no headroom beyond 65504: saturate instead of producing inf
  hi = __float2half_rn(x);
  lo = __float2half_rn(x - __half2float(hi));
}
// One-plane fp16 operand mode (emo_conv_desc.operand_fp16 with a_lo == w_lo == NULL): the plane is the hi plane of the split
// above, fp16(x * s) with the same saturation; one fp16 MMA per product, ~2^-11 relative per operand.
__device__ __forceinline__ __half f16_plane(float xs) { return __float2half_rn(fminf(fmaxf(xs, -65000.f), 65000.f)); }
__device__ __forceinline__ uint2 plane4_h(const float4& v, float s) {
  return make_uint2(pack_f16x2(f16_plane(v.x * s), f16_plane(v.y * s)), pack_f16x2(f16_plane(v.z * s), f16_plane(v.w * s)));
}
__device__ __forceinline__ void split4_h(const float4& v, float s, uint2& hi, uint2& lo) {
  __half h0, h1, h2, h3, l0, l1, l2, l3;
  split_f16(v.x * s, h0, l0);
  split_f16(v.y * s, h1, l1);
  split_f16(v.z * s, h2, l2);
  split_f16(v.w * s, h3, l3);
  hi.x = pack_f16x2(h0, h1);
  hi.y = pack_f16x2(h2, h3);
  lo.x = pack_f16x2(l0, l1);
  lo.y = pack_f16x2(l2, l3);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The video loop's foreground / background blend of one value (E_emo_infer_video.ipynb cell 41): m' = (m > thr ? m : 0)^8,
// m' * *img + (1 - m') * *bg.  composite_kernel and the bilinear taps of s2_prepare_composite_kernel both call it, so they give
// the same bits.
__device__ __forceinline__ float composite_pixel(float m, const float* img, const float* bg, float thr) {
  m = m > thr ? m : 0.f;
  const float m2 = m * m, m4 = m2 * m2, m8 = m4 * m4;
  return m8 * __ldg(img) + (1.f - m8) * __ldg(bg);
}

__device__ __forceinline__ float act_apply(float v, int act) {
  switch (act) {
    case EMO_ACT_RELU: return fmaxf(v, 0.f);
    case EMO_ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    case EMO_ACT_TANH: return tanhf(v);
    default: return v;
  }
}

}  // namespace emo
