/*
 * emoportraits_b200 — C-ABI of the H100-native (sm_90a) volumetric-avatar inference hot path.
 *
 * Drop-in boundary (SURVEY.md §8b): the reference has no FFI; its hot path is torch library
 * calls made from `notebooks/infer.py:355-647` (InferenceWrapper.forward) into
 * `networks/volumetric_avatar/*`.  Each entry point below replaces one family of those torch
 * call sites; the reference line it replaces is cited next to it.  A maintainer binds these
 * with ctypes exactly as emoportraits_b200/lib.py does (see INTEGRATION.md).
 *
 * Conventions
 *  - plain pointers and sizes only; every pointer is a DEVICE pointer unless stated;
 *  - `stream` is a cudaStream_t passed as void*;
 *  - activations are fp32, channels-last ([N][D][H][W][C], D==1 for 2-D), unless a field says
 *    otherwise; tensor-core operands are the same tensors split into two bf16 planes
 *    (hi = bf16(x), lo = bf16(x - hi)) so that three bf16 MMAs reproduce an fp32 product to
 *    ~2^-16 relative (see DESIGN.md "precision");
 *  - every function returns EMO_OK (0) or a negative error code; emo_last_error() returns the
 *    message of the last failure on the calling thread;
 *  - no function allocates device memory; workspaces are passed in.
 */
#ifndef EMOPORTRAITS_B200_H
#define EMOPORTRAITS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EMO_OK 0
#define EMO_ERR_INVALID (-1) /* bad argument / unsupported shape */
#define EMO_ERR_CUDA (-2)    /* CUDA runtime / driver error */
#define EMO_ERR_ARCH (-3)    /* not running on sm_90 */

enum { EMO_ACT_NONE = 0, EMO_ACT_RELU = 1, EMO_ACT_SIGMOID = 2, EMO_ACT_TANH = 3 };

const char* emo_last_error(void);
int emo_version(void); /* 111: emo_pose_desc.smooth_one_minus; 110: + emo_resample_u8, emo_mask_dilate; 109: + emo_s2_prepare_composite, emo_s2_masked_stem, emo_s2_finish_masked; 108: + emo_s2_prepare, emo_s2_finish; 107: + emo_stem_pack; 106: one-plane fp16 operands (emo_conv_desc, emo_apply_desc, emo_grid_sample3d_desc.plane_fp16,
                          emo_split_f16 with lo == NULL) and the EMO_CONV_KERNEL_H1_* kernels; 105: + emo_conv_plan; 104: + emo_composite; 103: emo_conv_desc.post; 102: + emo_u8_to_image, emo_image_to_u8, emo_resize_bicubic; 101: emo_pose_desc and emo_conv_desc gained trailing fields */
/* sm count, and cc major*10+minor of the current device */
int emo_device_info(int* sm_count, int* cc);

/* ------------------------------------------------------------------------------------------------
 * grid_sample 3-D: trilinear, padding_mode='zeros', align_corners=False.
 * Replaces: models/stage_1/volumetric_avatar/va.py:261-265 (Model.grid_sample -> F.grid_sample 5-D)
 *           and the affine grid build notebooks/infer.py:441-444, 583-588 (identity_grid_3d.bmm(theta^T))
 * when `theta` is given instead of `grid`.
 * ------------------------------------------------------------------------------------------------ */
typedef struct {
  const float* in; /* input volume */
  int in_layout;   /* 0: NCDHW (torch-contiguous, drop-in for F.grid_sample), 1: channels-last NDHWC */
  int N, C, Din, Hin, Win;
  const float* grid;  /* [N][Do][Ho][Wo][3] (x,y,z) or NULL */
  const float* theta; /* [N][3][4] row-major or NULL: grid = lattice(linspace(-1,1)) . theta^T (va.py:101-105) */
  int Dout, Hout, Wout;
  float* out;             /* fp32 output or NULL */
  void* out_hi;           /* optional bf16 split planes (same indexing as out) */
  void* out_lo;
  /* output element strides (in elements) for n, c, d, h, w. */
  long long os_n, os_c, os_d, os_h, os_w;
  void* out_lo2;          /* optional third bf16 plane (with out_hi/out_lo) */
  /* one-plane fp16 operand mode (see emo_conv_desc.operand_fp16): when plane_fp16 != 0, out_hi receives fp16(y * plane_scale)
   * (plane_scale a power of two) and out_lo / out_lo2 must be NULL. */
  int plane_fp16;
  float plane_scale;
} emo_grid_sample3d_desc;
int emo_grid_sample3d(const emo_grid_sample3d_desc* d, void* stream);

/* grid_sample 2-D, bilinear, zeros, align_corners=False, affine grid from theta [N][2][3]
 * over an identity lattice linspace(-1,1,Hout/Wout).
 * Replaces: networks/volumetric_avatar/expression_embedder.py:224-231 (align_warp + F.grid_sample).
 * in: NCHW fp32; out: channels-last [N][Hout][Wout][C_pad] fp32 with per-channel (x-mean)/std
 * (expression_embedder.py:441-445, ResNetWrapper.forward normalisation) when mean/std non-NULL.
 * Channels c >= C of the output are zero-filled. */
typedef struct {
  const float* in;
  int N, C, Hin, Win;
  const float* theta; /* [N][2][3] */
  int Hout, Wout;
  const float* mean; /* [C] or NULL */
  const float* std;  /* [C] or NULL */
  float* out;        /* [N][Hout][Wout][C_pad] */
  int C_pad;
  float* out_nchw;   /* optional un-normalised NCHW copy (source_img_align), or NULL */
} emo_grid_sample2d_affine_desc;
int emo_grid_sample2d_affine(const emo_grid_sample2d_affine_desc* d, void* stream);

/* F.interpolate(mode='bilinear', align_corners=False) NCHW -> channels-last [N][Ho][Wo][C_pad]
 * with optional per-channel normalisation.
 * Replaces: head_pose_regressor.py:24-25, identity_embedder.py:82-86. */
typedef struct {
  const float* in;
  int N, C, Hin, Win, Hout, Wout;
  const float* mean;
  const float* std;
  float* out;
  int C_pad;
} emo_resize_bilinear_desc;
int emo_resize_bilinear(const emo_resize_bilinear_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * GroupNorm pieces.  nn.GroupNorm(32, C, eps=1e-5) (networks/volumetric_avatar/utils.py:953,957),
 * AdaptiveGroupNorm (utils.py:302-325), eval-mode BatchNorm folded to the same affine form.
 *   stats:    double [N][G][2] = (sum, sum of squares) over (C/G) x spatial
 *   finalize: A[n][c] = rstd*gamma', B[n][c] = beta' - mean*rstd*gamma'
 *             gamma' = gamma (plain)  or gamma*(ada_w)  with beta' = beta*ada_w + ada_b (adaptive,
 *             ada_w = gamma+dw, ada_b = beta+db per sample: utils.py:994-995)
 *   apply:    y = act(x*A + B [+ res*A2 + B2]) -> fp32 and/or bf16 hi/lo planes, optional
 *             nearest x2 upsample on write (utils.py:685 F.interpolate(scale_factor=stride)).
 * ------------------------------------------------------------------------------------------------ */
int emo_gn_stats(const float* x, int N, long long spatial, int C, int G, double* stats, void* stream);

typedef struct {
  const double* stats; /* [N][G][2] */
  int N, C, G;
  double count;       /* elements per (n, group) */
  float eps;
  const float* gamma; /* [C] */
  const float* beta;  /* [C] */
  const float* ada_w; /* [N][C] or NULL */
  const float* ada_b; /* [N][C] or NULL */
  float* A;           /* [N][C] */
  float* B;           /* [N][C] */
} emo_gn_finalize_desc;
int emo_gn_finalize(const emo_gn_finalize_desc* d, void* stream);

typedef struct emo_apply_desc_s {
  const float* x; /* [N][S][C] fp32 channels-last, S = D*H*W */
  int N, C;
  int D, H, W;
  const float* A; /* [N][C] or NULL (identity) */
  const float* B;
  int ab_per_sample; /* 1: A,B are [N][C]; 0: [C] shared by all samples */
  const float* res;  /* optional residual, same shape as x */
  const float* A2;   /* optional affine on the residual [C] */
  const float* B2;
  int act;
  int up; /* 1 or 2: nearest upsample factor applied on H,W (D untouched) when writing */
  float* out;   /* optional fp32 [N][D][H*up][W*up][C] */
  void* out_hi; /* optional bf16 planes, same shape as out */
  void* out_lo;
  void* out_lo2; /* optional third plane (needs out_hi/out_lo) */
  /* fused GroupNorm finalisation (replaces A/B): when `stats` is given the kernel derives the per-(n,c) scale/shift
   * from the statistics itself (same arithmetic as emo_gn_finalize), saving a launch per normalisation. */
  const double* stats; /* [N][G][2] or NULL */
  int G;
  double count;
  float eps;
  const float* gamma; /* [C] */
  const float* beta;  /* [C] */
  const float* ada_w; /* [N][C] or NULL */
  const float* ada_b;
  /* fp16 two-plane operand mode (see emo_conv_desc.operand_fp16): when plane_fp16 != 0, out_hi/out_lo receive the fp16
   * planes of y * plane_scale (plane_scale a power of two that keeps the planes in fp16's normal range; out_lo2 unused).
   * With out_lo == NULL only out_hi is written: the one-plane fp16 operand fp16(y * plane_scale). */
  int plane_fp16;
  float plane_scale;
} emo_apply_desc;
int emo_apply(const emo_apply_desc* d, void* stream);

/* Fused image head: out[n][o][s] = act_out( bias[o] + sum_c w[o][c] * relu(GN(x)[n][s][c]) ), Cout <= 4, NCHW output.
 * Replaces the tail of ImageDecoder (decoder.py:398-410: dec_img_head = norm -> ReLU -> 1x1 Conv2d_ws -> sigmoid, applied at
 * decoder.py:238): one pass over the 512^2 x 128 fp32 tensor in exact fp32 instead of a GN-apply pass writing bf16 planes
 * plus a 3-channel tensor-core conv.  GroupNorm scale/shift are derived from `stats` in the kernel (as in emo_apply). */
typedef struct {
  const float* x; /* [N][S][C] fp32 channels-last */
  int N, C;
  long long S;         /* spatial positions per sample */
  const double* stats; /* [N][G][2] */
  int G;
  double count;
  float eps;
  const float* gamma; /* [C] */
  const float* beta;  /* [C] */
  const float* w;     /* [Cout][C] fp32 (already folded: weight standardisation / spectral norm) */
  const float* bias;  /* [Cout] or NULL */
  int Cout;           /* 1..4 */
  int act_out;        /* EMO_ACT_* applied to the head output */
  float* out;         /* [N][Cout][S] fp32 */
} emo_gn_head_desc;
int emo_gn_head(const emo_gn_head_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Implicit-GEMM convolution on wgmma (2-D and 3-D, any kernel extent per dim — the path uses 1, 3 and the folded
 * 4x4 stride-2 form of `3x3 conv -> 2x2 avgpool` —, stride 1 or 2, zero padding), bf16x2-split operands, fp32
 * accumulation in registers.
 * Replaces: F.conv2d / F.conv3d call sites of utils.py:661-788 (ResBlock), :894-915 (Conv*_ws),
 *           decoder.py:77-81,349-356, local_encoder.py:104-108, warp_generator_resnet.py:99-106.
 * ------------------------------------------------------------------------------------------------ */
typedef struct {
  const void* a_hi; /* activations, bf16 channels-last [N][Din][Hin][Win][Cin] */
  const void* a_lo;
  int N, Din, Hin, Win, Cin;
  const void* w_hi; /* weights, bf16 [taps][Cout_pad][Cin], taps ordered (kd,kh,kw) */
  const void* w_lo;
  int Cout, Cout_pad;
  int kd, kh, kw;
  int sd, sh, sw;    /* strides */
  int pd, ph, pw;    /* paddings */
  int Dout, Hout, Wout;
  const float* bias;     /* [Cout] or NULL */
  const float* residual; /* fp32 channels-last [N][Dout>>rs_d][Hout>>rs][Wout>>rs][Cout] or NULL */
  int res_shift;         /* residual is read at (h>>res_shift, w>>res_shift) (nearest-upsampled skip) */
  int act;               /* applied after bias+residual */
  const float* post_add; /* added after the activation, [Dout][Hout][Wout][Cout] (shared by all n) or NULL */
  float* out;            /* fp32 */
  int out_nchw;          /* 0: channels-last; 1: [N][Cout][Dout][Hout][Wout] */
  double* stats;         /* optional GN statistics of the output: [N][G][2] accumulated (+=) */
  int G;
  /* optional third bf16 plane of both operands (lo2 = bf16(x - hi - lo)): six MMAs per product, ~2^-24 relative
   * (fp32-faithful) for the numerically sensitive embedding / warp networks.  Both or neither. */
  const void* a_lo2;
  const void* w_lo2;
  /* MMAs accumulated in one wgmma register chunk before it is added to the fp32 sums (0 = default 24).  The tensor core
   * accumulates with truncation; short chunks keep that bias ~1e-6 relative (DESIGN.md "precision"). */
  int acc_chunk_mmas;
  /* optional split-K workspace: fp32, >= 2*N*Dout*Hout*Wout*Cout elements, no initial state needed.  When given, layers
   * with too few tiles to fill the machine split their K loop over CTAs (each part stores its partial sums to its own slice
   * of N*Dout*Hout*Wout*Cout elements, then one finalize launch sums the slices in part order and applies
   * bias/residual/activation/statistics; the workspace is not written back).  NULL: never split. */
  float* splitk_ws;
  long long splitk_ws_elems;
  /* sub-pixel evaluation of `nearest x2 -> 3x3 conv` (ImageDecoder up blocks, decoder.py:241-358 / utils.py:761-788 with
   * upsample): when non-zero, a_hi/a_lo are the LOW-resolution planes [N][1][Hin][Win][Cin], Hout = 2 Hin, Wout = 2 Win,
   * kd,kh,kw = 1,3,3 / pad 0,1,1 describe the convolution being replaced, and w_hi/w_lo hold the phase-folded weights
   * [16 = 4 output phases x 2x2 taps][Cout_pad][Cin]: a 3x3 conv over a nearest-upsampled map is, per output-pixel parity,
   * a 2x2 conv over the low-resolution map (4/9 of the MMAs, no upsampled operand in HBM).  residual/res_shift/post_add
   * are indexed at the output resolution as usual.  Two-plane operands only. */
  int upconv;
  /* fp16 two-plane operand mode: a_hi/a_lo and w_hi/w_lo are FP16 planes of (activation * sa) and (weight * sw), sa and sw
   * powers of two chosen by the caller (emo_apply.plane_scale / the weight packer); the kernel issues the same three MMAs
   * (hi*hi + hi*lo + lo*hi, kind::f16 with fp16 inputs) and multiplies the fp32 sums by out_scale = 1 / (sa * sw) before
   * bias / residual.  ~22 mantissa bits per operand: fp32-faithful like the three-plane bf16 mode at half its MMAs.
   * Not combinable with a_lo2/w_lo2 or upconv.
   * One-plane fp16 operands: operand_fp16 with a_lo == w_lo == NULL (and no a_lo2/w_lo2).  a_hi / w_hi are fp16(activation * sa)
   * and fp16(weight * sw); ONE MMA per product (~2^-11 relative per operand: decoder-only, DESIGN.md section 2).  Also
   * combinable with upconv (w_hi then holds the phase-folded weights). */
  int operand_fp16;
  float out_scale;
  /* optional post-op on the convolution's output: y = act(GN-or-affine(out) [+ res*A2 + B2]) -> fp32 and/or operand planes,
   * exactly emo_apply with x = out (post->x is ignored; a GroupNorm post-op must name the convolution's own statistics:
   * post->stats == stats; up must be 1).  Small split-K layers (<= 64 Ki elements per sample) run it inside the finalize
   * step - one launch instead of finalize + emo_apply, `out` is then NOT written - every other layer runs emo_apply after
   * the convolution.  NULL: none. */
  const struct emo_apply_desc_s* post;
} emo_conv_desc;
int emo_conv_igemm(const emo_conv_desc* d, void* stream);

/* The launch plan emo_conv_igemm picks for a descriptor on a device with `sm_count` SMs.  Host arithmetic only: no CUDA
 * call, no device needed, pointers are checked (null, alignment) but never dereferenced.  Runs the same argument checks
 * and returns the same error codes as emo_conv_igemm. */
enum {
  /* conv_igemm_kernel<KC, NP, PS (sub-pixel form), F16 (fp16 operands)> */
  EMO_CONV_KERNEL_BF16X2_KC64 = 0, /* conv_igemm_kernel<64, 2, false, false> */
  EMO_CONV_KERNEL_BF16X2_KC32 = 1, /* conv_igemm_kernel<32, 2, false, false> */
  EMO_CONV_KERNEL_BF16X3_KC64 = 2, /* conv_igemm_kernel<64, 3, false, false> */
  EMO_CONV_KERNEL_BF16X3_KC32 = 3, /* conv_igemm_kernel<32, 3, false, false> */
  EMO_CONV_KERNEL_F16_KC64 = 4,    /* conv_igemm_kernel<64, 2, false, true> */
  EMO_CONV_KERNEL_F16_KC32 = 5,    /* conv_igemm_kernel<32, 2, false, true> */
  EMO_CONV_KERNEL_UPCONV_KC64 = 6, /* conv_igemm_kernel<64, 2, true, false> */
  /* one-plane fp16 operands (operand_fp16 with a_lo == w_lo == NULL), reported with NP = 1; ids 7, 8, 9 */
  EMO_CONV_KERNEL_H1_KC64,         /* conv_igemm_kernel<64, 1, false, true> */
  EMO_CONV_KERNEL_H1_KC32,         /* conv_igemm_kernel<32, 1, false, true> */
  EMO_CONV_KERNEL_H1_UPCONV_KC64   /* conv_igemm_kernel<64, 1, true, true> */
};
enum {
  EMO_CONV_FINISH_NONE = 0,           /* the convolution kernel writes the output */
  EMO_CONV_FINISH_FINALIZE = 1,       /* split-K: the finalize kernel sums the parts */
  EMO_CONV_FINISH_POST = 2,           /* split-K with a post-op: one cluster kernel sums, normalises and writes the post-op */
  EMO_CONV_FINISH_FINALIZE_APPLY = 3, /* split-K: finalize, then emo_apply runs the post-op */
  EMO_CONV_FINISH_APPLY = 4           /* un-split with a post-op: emo_apply after the convolution kernel */
};
typedef struct {
  int kernel;            /* EMO_CONV_KERNEL_* */
  int KC, NP, fp16;      /* channels per k-chunk, operand planes, fp16 operands */
  int BN;                /* N tile (output channels per tile) */
  int ksplit;            /* K parts (1: not split) */
  int yreuse, sa, sb;    /* row-reuse main loop, its A (halo tile) and B ring depths */
  int stages;            /* pipeline stages (the B ring depth with row reuse) */
  int flush;             /* k-steps per accumulation chunk */
  int tw, th, td;        /* pixel box of one tile */
  int m_tiles, n_tiles;  /* pixel tiles, N tiles (x4 output phases with upconv) */
  int grid;              /* CTAs launched: min(m_tiles * n_tiles * ksplit, sm_count) */
  int finish;            /* EMO_CONV_FINISH_* */
} emo_conv_plan_info;
int emo_conv_plan(const emo_conv_desc* d, int sm_count, emo_conv_plan_info* out);

/* Direct fp32 SIMT convolution for the layers the tensor-core path does not take (Cin not a
 * multiple of 32: the RGB stems local_encoder.py:66-74 7x7 and torchvision resnet conv1).
 * x: fp32 channels-last [N][Hin][Win][Cin_pad]; w: fp32 [kh][kw][Cin_pad][Cout]. */
typedef struct {
  const float* x;
  int N, Hin, Win, Cin_pad;
  const float* w;
  int Cout, kh, kw, stride, pad;
  int Hout, Wout;
  const float* bias;
  float* out; /* fp32 channels-last */
  double* stats;
  int G;
} emo_conv_direct_desc;
int emo_conv_direct(const emo_conv_direct_desc* d, void* stream);

/* The 7x7 RGB stem as a tensor-core operand (stage-2 fast mode): the 7 horizontal taps of each pixel become 28 channels of one
 * fp16 plane, so that the stem runs on emo_conv_igemm as a 7x1 convolution over Cin = 32 (pad (3, 0)).
 * x: fp32 channels-last [N][H][W][C], C == 4 (the padded RGB of emo_resize_bilinear), 16-byte aligned.
 * out: fp16 [N][H][W][32], 16-byte aligned:  out[n][h][w][kx*4 + c] = fp16(scale * x[n][h][w + kx - 3][c]) for kx = 0..6,
 *      exactly 0 for columns outside the image and for channels 28..31. */
int emo_stem_pack(const float* x, int N, int H, int W, int C, float scale, void* out, void* stream);

/* y[m][n] = act((sum_k x[m][k] * w[n][k] + bias[n] + add[m][n]) * scale), fp32 SIMT.
 * Replaces: va.py:820-823 (pose_unsqueeze_nw), :855 (warp_embed_head_orig_nw on a 4x4 map),
 *           utils.py:1146 (ProjectorNorm u.E.v), warp_generator_resnet.py:138 (first_conv),
 *           expression_embedder.py:455-460 (pose_head), resnet fc layers.
 * Output element (m, n) is written at out[m*os_m + n*os_n]. */
typedef struct {
  const float* x;
  long long xs_m, xs_k; /* element strides of x */
  const float* w;       /* [N][K] row-major */
  const float* bias;    /* [N] or NULL */
  const float* add;     /* same indexing as out, or NULL */
  float scale;
  int act;
  int M, N, K;
  float* out;
  long long os_m, os_n;
} emo_linear_desc;
int emo_linear(const emo_linear_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Resampling on channels-last fp32 tensors.
 * trilinear: F.interpolate(mode='trilinear', scale_factor=(fd,fh,fw)), align_corners=False
 *            (unet_3d.py:224,273-275, warp_generator_resnet.py:160-163); optional `add` tensor of
 *            the output shape (unet_3d.py:286 `outputs + outputs_skip`); optional GN stats of the result.
 * avgpool:   AvgPool2d/3d with kernel == stride (utils.py:964-969, unet_3d.py:87-90,193, warp_generator_resnet.py:115)
 * maxpool:   torchvision resnet maxpool 3x3 s2 p1.
 * ------------------------------------------------------------------------------------------------ */
typedef struct {
  const float* x;
  int N, D, H, W, C;
  int fd, fh, fw; /* 1 or 2 */
  const float* add;
  float* out;
  double* stats;
  int G;
} emo_resample_desc;
int emo_upsample_trilinear(const emo_resample_desc* d, void* stream);
int emo_avgpool(const emo_resample_desc* d, void* stream);
int emo_maxpool2d_3x3s2(const float* x, int N, int H, int W, int C, float* out, void* stream);
/* mean over spatial positions: [N][S][C] -> [N][C] */
int emo_global_avgpool(const float* x, int N, long long S, int C, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Pose algebra on device (removes the per-frame host sync of infer.py:568-569, 699-736).
 *   srt [N][9] = (scale xyz, yaw pitch roll, translation xyz) from the head-pose regressor, or from the caller's
 *             custome_target_theta_embed (infer.py:566-567)
 *   theta = S.R.T (utils/point_transforms.py:187-240), or theta_in when given
 *   mix != 0: get_mixing_theta(source_theta, theta) (infer.py:686-736): polar decompositions in fp64
 *             (scipy.linalg.polar), result rows [:3]; mix_old selects the product of :727 (1) or :729 (0)
 *   smooth_state != NULL: smooth_pose=True (infer.py:571-581): state = theta_n * momentum + state * smooth_one_minus
 *             (each product rounded to fp32, then the sum) on rows [:3], sample after sample in order, the state
 *             (self.theta) carried across calls in smooth_state [3][4]; smooth_init != 0 seeds the state with the first
 *             sample's theta (self.theta is None)
 *   outputs: theta_out [N][4][4]; theta_warp [N][3][4] = (invert ? inverse(theta) : theta)[:3]
 *            (infer.py:443 / :586); align2d [N][2][3] = (inverse(theta4)[[0,1,3]][:, [0,1,3]] . diag(.5,.5,1))[:2]
 *            (expression_embedder.py:176-203).
 * ------------------------------------------------------------------------------------------------ */
typedef struct {
  const float* srt;          /* [N][9], or NULL when theta_in is given */
  const float* source_theta; /* [4][4] or NULL (required when mix) */
  int N;
  int mix;
  int invert_warp;
  float* theta_out;  /* [N][4][4] */
  float* theta_warp; /* [N][3][4] */
  float* align2d;    /* [N][2][3] */
  const float* theta_in; /* [N][4][4] or NULL: start from this theta instead of S.R.T(srt) */
  int mix_old;           /* with mix: 1 = translation_t . rotation_t . stretch_s (infer.py:727) */
  int smooth_init;       /* with smooth_state: 1 = seed the state with sample 0's theta first */
  float* smooth_state;   /* [3][4] or NULL */
  float smooth_momentum; /* pose_momentum (infer.py:64, default 0.5) */
  float smooth_one_minus; /* with smooth_state: 1 - pose_momentum as Python computes it (in double, from the unrounded
                             momentum) rounded to fp32, the factor torch applies to the state; it is not a function of
                             the fp32 smooth_momentum (0.9 gives 0.1f, 1 - 0.9f rounds 3 ulp above it).  0: not
                             given, 1 - smooth_momentum in fp32 (a descriptor from before version 111) */
} emo_pose_desc;
int emo_pose_theta(const emo_pose_desc* d, void* stream);

/* fp32 -> bf16 hi/lo(/lo2) planes (n elements); lo2 may be NULL. */
int emo_split_bf16(const float* x, long long n, void* hi, void* lo, void* lo2, void* stream);
/* fp32 -> fp16 hi/lo planes of x * scale (n elements), the operand format of emo_conv_desc.operand_fp16.  lo == NULL: the
 * one-plane operand fp16(x * scale) only. */
int emo_split_f16(const float* x, long long n, float scale, void* hi, void* lo, void* stream);
/* ------------------------------------------------------------------------------------------------
 * Pre/post-processing at the wrapper boundary (SURVEY.md §8f-2).
 *   emo_u8_to_image   uint8 [N][H][W][C] (PIL / numpy layout) -> fp32 [N][C][H][W] = u / 255
 *                     replaces transforms.ToTensor() in notebooks/infer.py:229-243 (convert_to_tensor)
 *   emo_image_to_u8   fp32 [N][C][H][W] -> uint8 [N][H][W][C] = trunc(clamp(x, 0, 1) * 255)
 *                     replaces `.clamp(0, 1)` + transforms.ToPILImage() (mul(255).byte()) notebooks/infer.py:641-644;
 *                     a NaN pixel becomes 0 (torch's clamp keeps the NaN, whose byte conversion is undefined)
 *   emo_resize_bicubic fp32 [N][C][Hin][Win] -> [N][C][Hout][Wout]: F.interpolate(mode='bicubic', align_corners=False),
 *                     A = -0.75, border-replicated taps; replaces notebooks/infer.py:399-403, 551-556
 * ------------------------------------------------------------------------------------------------ */
int emo_u8_to_image(const unsigned char* nhwc, int N, int H, int W, int C, float* nchw, void* stream);
int emo_image_to_u8(const float* nchw, int N, int C, int H, int W, unsigned char* nhwc, void* stream);
int emo_resize_bicubic(const float* in, int N, int C, int Hin, int Win, int Hout, int Wout, float* out, void* stream);
/* The stage-1 -> stage-2 handoff of a refined frame (notebooks/infer_s2.py:351-376 on the stage-1 image), one pass each side.
 *   emo_s2_prepare  img fp32 [N][3][Hin][Win] -> resized fp32 [N][3][S][S], the bilinear resize (align_corners=False) with the
 *                   bits of emo_resize_bilinear, and the stage-2 stem's operand, exactly one of:
 *                     x4     fp32 [N][S][S][4] = (R, G, B, 0), emo_resize_bilinear's output with C_pad 4 (the exact mode's
 *                            emo_conv_direct input), 16-byte aligned;
 *                     plane  fp16 [N][S][S][32], emo_stem_pack's plane of that x4 with scale plane_scale > 0 (the fast mode's
 *                            7x1 implicit-GEMM operand), 16-byte aligned.
 *   emo_s2_finish   resized, add fp32 [N][3][H][W] -> out fp32 [N][3][H][W] = clamp(resized + add, 0, 1) (one fp32 add, a NaN
 *                   stays NaN, as torch's clamp) and u8 uint8 [N][H][W][3], emo_image_to_u8 of out. */
int emo_s2_prepare(const float* img, int N, int Hin, int Win, int S, float* resized, float* x4, void* plane, float plane_scale,
                   void* stream);
int emo_s2_finish(const float* resized, const float* add, int N, int H, int W, float* out, unsigned char* u8, void* stream);
/* The same handoff with the stage-2 masks of notebooks/infer_s2.py:356-376 and the video loop's composite (E_emo_infer_video.ipynb
 * cell 41), each bit for bit the eager composition it replaces:
 *   emo_s2_prepare_composite  emo_s2_prepare of emo_composite(img, matte, bg, threshold) (img fp32 [N][3][Hin][Win], matte fp32
 *                             [N][1][Hin][Win], bg fp32 [3][Hin][Win]); the composited image never exists in memory.  At most one
 *                             stem operand: none when the stem reads a masked operand (emo_s2_masked_stem).
 *   emo_s2_masked_stem        the stem's operand of resized * matte (resized fp32 [N][3][S][S], matte fp32 [N][1][S][S]):
 *                             exactly one of x4 (R m, G m, B m, 0 m) fp32 [N][S][S][4] or emo_stem_pack's plane of that x4,
 *                             16-byte aligned.
 *   emo_s2_finish_masked      emo_s2_finish with the residual masked: out = clamp(resized + add * (matte * face), 0, 1), one fp32
 *                             rounding per operation, a NaN stays NaN; matte fp32 [N][1][H][W], face uint8 0 / 1 [N][1][H][W] (the
 *                             first mask of emo_parsing_masks) or NULL for matte alone; u8 as emo_s2_finish. */
int emo_s2_prepare_composite(const float* img, const float* matte, const float* bg, float threshold, int N, int Hin, int Win, int S,
                             float* resized, float* x4, void* plane, float plane_scale, void* stream);
int emo_s2_masked_stem(const float* resized, const float* matte, int N, int S, float* x4, void* plane, float plane_scale, void* stream);
int emo_s2_finish_masked(const float* resized, const float* add, const float* matte, const unsigned char* face, int N, int H, int W,
                         float* out, unsigned char* u8, void* stream);
/* Foreground / background compositing of the video loop (notebooks/E_emo_infer_video.ipynb cell 41, connect_img_and_bg):
 *   m' = (mask > threshold ? mask : 0)^8;  out = m' * img + (1 - m') * bg
 * img, out fp32 [N][C][H][W]; mask fp32 [N][1][H][W]; bg fp32 [C][H][W] (one background for the whole clip). */
int emo_composite(const float* img, const float* mask, const float* bg, int N, int C, int H, int W, float threshold, float* out, void* stream);
/* ------------------------------------------------------------------------------------------------
 * Mask pre/post-processing around the EXTERNAL mask networks (BiSeNet face parsing, MODNet matting: separate checkouts that
 * are not part of the reference tree).  All tensors fp32 NCHW on the device unless noted.
 *   emo_parsing_prepare  out[n][c] = bilinear_resize((in[n][c] - mean[c]) / std[c], Hout x Wout), align_corners=False
 *                        replaces networks/volumetric_avatar/face_parcing.py:57-58 (normalise, F.interpolate to 512 x 512)
 *   emo_parsing_masks    logits [N][K][Hin][Win] -> bilinear resize to Hout x Wout -> argmax over K -> membership of the label
 *                        in four class sets; out uint8 [4][N][Hout][Wout] (0/1), labels uint8 [N][Hout][Wout] or NULL.
 *                        label_sets: HOST array of four 32-bit sets (bit k = class k).  K <= 32.
 *                        replaces face_parcing.py:60-80 (F.interpolate, argmax, the four `mask += labels == i` loops)
 *   emo_resize_area      out = adaptive_average_pool(in * scale + shift, Hout x Wout) = F.interpolate(mode='area')
 *                        replaces notebooks/infer.py:651-657 + :676 (Normalize(0.5, 0.5) then area resize) and :682
 * ------------------------------------------------------------------------------------------------ */
int emo_parsing_prepare(const float* in, int N, int C, int Hin, int Win, int Hout, int Wout, const float* mean, const float* std,
                        float* out, void* stream);
int emo_parsing_masks(const float* logits, int N, int K, int Hin, int Win, int Hout, int Wout, const unsigned* label_sets,
                      unsigned char* out, unsigned char* labels, void* stream);
int emo_resize_area(const float* in, int N, int C, int Hin, int Win, int Hout, int Wout, float scale, float shift, float* out,
                    void* stream);
/* ------------------------------------------------------------------------------------------------
 * Image plumbing of the demo video loop (E_emo_infer_video.ipynb cells 40, 46-49)
 *   emo_resample_u8  Pillow's Image.crop((x0, y0, x0 + crop_w, y0 + crop_h)).resize((out_w, out_h), f), bit for bit, for an
 *                    interleaved 3-channel uint8 image (LANCZOS or BICUBIC: the filter lives in the taps).  src [src_h] rows
 *                    of src_pitch bytes, dst [out_h] rows of dst_pitch bytes (a column offset is a pointer offset); *_bgr
 *                    give each side's channel order, so a BGR frame is read and a BGR video row written directly.  Pixels
 *                    outside the source read as 0 (Image.crop's padding).  h_taps / v_taps: per output column / row, one
 *                    row of (2 + kmax) ints: first tap in crop coordinates, tap count, then the coefficients with 22
 *                    fractional bits (Pillow's precompute_coeffs + normalize_coeffs_8bpc); NULL exactly for an axis whose
 *                    size does not change (Pillow skips that pass; with both NULL the call is a copy).  With both passes
 *                    the horizontal one writes crop rows tmp_y0 .. tmp_y0 + tmp_rows (the rows the vertical taps read) to
 *                    tmp [tmp_rows][out_w][3].  replaces the PIL resizes of cells 46-49.
 *   emo_mask_dilate  out = max over the (2 radius + 1)^2 window, clipped to the image, of (m >= thr); m, out fp32
 *                    [N][H][W], out 0 / 1, tmp uint8 [N][H][W].  replaces cell 40's cv2.dilate((m >= 0.8), ones(21, 21),
 *                    iterations=2) (radius 20).
 * ------------------------------------------------------------------------------------------------ */
int emo_resample_u8(const unsigned char* src, int src_h, int src_w, long long src_pitch, int src_bgr, int x0, int y0, int crop_w,
                    int crop_h, unsigned char* dst, int out_h, int out_w, long long dst_pitch, int dst_bgr, const int* h_taps,
                    int h_kmax, const int* v_taps, int v_kmax, unsigned char* tmp, int tmp_y0, int tmp_rows, void* stream);
int emo_mask_dilate(const float* m, int N, int H, int W, float thr, int radius, unsigned char* tmp, float* out, void* stream);
/* L2 flush helpers for benchmarks: emo_l2_flush writes `bytes` of `buf` (L2 is left full of DIRTY foreign lines: the next
 * kernel also pays for their write-back); emo_l2_flush_clean writes and then reads the buffer back (L2 is left full of
 * CLEAN foreign lines). */
int emo_l2_flush(void* buf, long long bytes, void* stream);
int emo_l2_flush_clean(void* buf, long long bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* EMOPORTRAITS_B200_H */
