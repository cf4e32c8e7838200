// Image plumbing of the demo notebook's video loop (E_emo_infer_video.ipynb cells 40, 46-49), on the device:
//
//   emo_resample_u8  Pillow's `Image.crop(box).resize(size, f)` of an interleaved 3-channel uint8 image, bit for bit, for the
//                    integer boxes and the two filters (LANCZOS, BICUBIC) the notebook uses.  The filter taps are Pillow's
//                    fixed-point coefficients (22 fractional bits), computed on the host (ops.resample_taps) and read here; each
//                    pass sums pixel * k in int32 from 1 << 21, shifts right by 22 and clips to [0, 255], as
//                    libImaging/Resample.c does.  The horizontal pass runs first, into a uint8 intermediate of the rows the
//                    vertical pass reads.  Pixels outside the source read as 0 (Image.crop's padding).
//   emo_mask_dilate  max over a (2r+1)^2 window, clipped to the image, of (m >= thr): cell 40's
//                    cv2.dilate((m >= 0.8).float(), ones(21, 21), iterations=2) is r = 20.  Two separable passes.
#include "common.cuh"

namespace emo {

constexpr int RS_BITS = 22;  // Pillow's PRECISION_BITS (32 - 8 - 2)

enum { RS_HORIZONTAL = 0, RS_VERTICAL = 1, RS_COPY = 2 };

// Pillow's crop padding: a pixel outside the source reads as 0
__device__ __forceinline__ int rs_pixel(const unsigned char* __restrict__ src, int sh, int sw, long long pitch, int y, int x, int c) {
  return (y >= 0 && y < sh && x >= 0 && x < sw) ? (int)__ldg(src + (long long)y * pitch + 3 * x + c) : 0;
}

__device__ __forceinline__ unsigned char rs_clip8(int acc) {
  const int v = acc >> RS_BITS;  // arithmetic shift: floor, as Pillow's clip8 lookup
  return (unsigned char)(v < 0 ? 0 : v > 255 ? 255 : v);
}

// One pass over an (oh, ow) output: MODE RS_HORIZONTAL filters source row oy + y along x, RS_VERTICAL source column ox + x along
// y, RS_COPY reads pixel (oy + y, ox + x).  taps: one row of (2 + kmax) ints per output index along the filtered axis:
// first tap (relative to the origin), tap count, then the coefficients.  swap: the destination's channel order is the reverse
// of the source's (RGB <-> BGR).
template <int MODE>
__global__ void resample_u8_kernel(const unsigned char* __restrict__ src, int sh, int sw, long long spitch, int ox, int oy,
                                   unsigned char* __restrict__ dst, int oh, int ow, long long dpitch, int swap,
                                   const int* __restrict__ taps, int kmax) {
  const long long total = (long long)oh * ow;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(t % ow), y = (int)(t / ow);
    int acc[3];
    if (MODE == RS_COPY) {
      for (int c = 0; c < 3; ++c) acc[c] = rs_pixel(src, sh, sw, spitch, oy + y, ox + x, c);
    } else {
      const int* tp = taps + (long long)(MODE == RS_HORIZONTAL ? x : y) * (2 + kmax);
      const int first = __ldg(tp), n = __ldg(tp + 1);
      for (int c = 0; c < 3; ++c) acc[c] = 1 << (RS_BITS - 1);
      for (int j = 0; j < n; ++j) {
        const int k = __ldg(tp + 2 + j);
        const int sy = MODE == RS_HORIZONTAL ? oy + y : oy + first + j;
        const int sx = MODE == RS_HORIZONTAL ? ox + first + j : ox + x;
        for (int c = 0; c < 3; ++c) acc[c] += rs_pixel(src, sh, sw, spitch, sy, sx, c) * k;
      }
      for (int c = 0; c < 3; ++c) acc[c] = rs_clip8(acc[c]);
    }
    unsigned char* d = dst + (long long)y * dpitch + 3 * x;
    d[0] = (unsigned char)(swap ? acc[2] : acc[0]);  // selects, not an indexed load: acc stays in registers
    d[1] = (unsigned char)acc[1];
    d[2] = (unsigned char)(swap ? acc[0] : acc[2]);
  }
}

// VERT = false: tmp[n][y][x] = any(m[n][y][x - r .. x + r] >= thr); VERT = true: out[n][y][x] = any(tmp[n][y - r .. y + r][x])
template <bool VERT>
__global__ void mask_dilate_kernel(const float* __restrict__ m, const unsigned char* __restrict__ tmp_in, int N, int H, int W,
                                   float thr, int r, unsigned char* __restrict__ tmp_out, float* __restrict__ out) {
  const long long total = (long long)N * H * W;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(t % W);
    const long long ny = t / W;
    const int y = (int)(ny % H);
    const long long plane = (ny / H) * H * W;
    bool hit = false;
    if (!VERT) {
      const float* row = m + plane + (long long)y * W;
      for (int xx = max(x - r, 0); xx <= min(x + r, W - 1) && !hit; ++xx) hit = __ldg(row + xx) >= thr;
      tmp_out[t] = hit ? 1 : 0;
    } else {
      const unsigned char* col = tmp_in + plane + x;
      for (int yy = max(y - r, 0); yy <= min(y + r, H - 1) && !hit; ++yy) hit = __ldg(col + (long long)yy * W) != 0;
      out[t] = hit ? 1.f : 0.f;
    }
  }
}

static inline unsigned grid_for(long long total, int block, int cap) {
  const long long b = cdivll(total, block);
  return (unsigned)(b < 1 ? 1 : b > cap ? cap : b);
}

template <int MODE>
static int resample_pass(const unsigned char* src, int sh, int sw, long long spitch, int ox, int oy, unsigned char* dst, int oh, int ow,
                         long long dpitch, int swap, const int* taps, int kmax, cudaStream_t stream) {
  launch_kernel(resample_u8_kernel<MODE>, grid_for((long long)oh * ow, 256, 132 * 16), 256, 0, stream, src, sh, sw, spitch, ox, oy, dst,
                oh, ow, dpitch, swap, taps, kmax);
  return check_launch("emo_resample_u8");
}

}  // namespace emo

using namespace emo;

extern "C" int emo_resample_u8(const unsigned char* src, int src_h, int src_w, long long src_pitch, int src_bgr, int x0, int y0,
                               int crop_w, int crop_h, unsigned char* dst, int out_h, int out_w, long long dst_pitch, int dst_bgr,
                               const int* h_taps, int h_kmax, const int* v_taps, int v_kmax, unsigned char* tmp, int tmp_y0,
                               int tmp_rows, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(src && dst, "emo_resample_u8: null pointer");
  EMO_REQUIRE(src_h > 0 && src_w > 0 && crop_w > 0 && crop_h > 0 && out_h > 0 && out_w > 0,
              "emo_resample_u8: bad shape (source %dx%d, crop %dx%d, output %dx%d)", src_w, src_h, crop_w, crop_h, out_w, out_h);
  EMO_REQUIRE(src_pitch >= 3ll * src_w && dst_pitch >= 3ll * out_w, "emo_resample_u8: a row pitch is smaller than its row");
  EMO_REQUIRE(!h_taps == (out_w == crop_w) && !v_taps == (out_h == crop_h),
              "emo_resample_u8: give taps exactly for each axis whose size changes (crop %dx%d -> %dx%d)", crop_w, crop_h, out_w, out_h);
  EMO_REQUIRE((!h_taps || h_kmax > 0) && (!v_taps || v_kmax > 0), "emo_resample_u8: taps need kmax > 0");
  EMO_REQUIRE(!(h_taps && v_taps) || (tmp && tmp_rows > 0 && tmp_y0 >= 0 && tmp_y0 + tmp_rows <= crop_h),
              "emo_resample_u8: two passes need the intermediate rows (tmp_y0 %d, tmp_rows %d of %d)", tmp_y0, tmp_rows, crop_h);
  const int swap = (src_bgr != 0) != (dst_bgr != 0);
  if (h_taps && v_taps) {
    const int rc = resample_pass<RS_HORIZONTAL>(src, src_h, src_w, src_pitch, x0, y0 + tmp_y0, tmp, tmp_rows, out_w, 3ll * out_w, 0,
                                                h_taps, h_kmax, stream);
    if (rc != EMO_OK) return rc;
    return resample_pass<RS_VERTICAL>(tmp, tmp_rows, out_w, 3ll * out_w, 0, -tmp_y0, dst, out_h, out_w, dst_pitch, swap, v_taps, v_kmax,
                                      stream);
  }
  if (h_taps)
    return resample_pass<RS_HORIZONTAL>(src, src_h, src_w, src_pitch, x0, y0, dst, out_h, out_w, dst_pitch, swap, h_taps, h_kmax, stream);
  if (v_taps)
    return resample_pass<RS_VERTICAL>(src, src_h, src_w, src_pitch, x0, y0, dst, out_h, out_w, dst_pitch, swap, v_taps, v_kmax, stream);
  return resample_pass<RS_COPY>(src, src_h, src_w, src_pitch, x0, y0, dst, out_h, out_w, dst_pitch, swap, nullptr, 0, stream);
}

extern "C" int emo_mask_dilate(const float* m, int N, int H, int W, float thr, int radius, unsigned char* tmp, float* out, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  EMO_REQUIRE(m && tmp && out, "emo_mask_dilate: null pointer");
  EMO_REQUIRE(N > 0 && H > 0 && W > 0 && radius >= 0, "emo_mask_dilate: bad shape (N=%d H=%d W=%d radius=%d)", N, H, W, radius);
  const long long total = (long long)N * H * W;
  launch_kernel(mask_dilate_kernel<false>, grid_for(total, 256, 132 * 16), 256, 0, stream, m, (const unsigned char*)nullptr, N, H, W, thr,
                radius, tmp, (float*)nullptr);
  const int rc = check_launch("emo_mask_dilate");
  if (rc != EMO_OK) return rc;
  launch_kernel(mask_dilate_kernel<true>, grid_for(total, 256, 132 * 16), 256, 0, stream, (const float*)nullptr, (const unsigned char*)tmp,
                N, H, W, thr, radius, (unsigned char*)nullptr, out);
  return check_launch("emo_mask_dilate");
}
