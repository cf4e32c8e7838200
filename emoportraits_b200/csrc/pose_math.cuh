// Pose algebra of the driver/source pass, one sample per call (a few hundred flops).  Host+device source: the CUDA
// kernel `pose_theta_kernel` (misc.cu) calls pose_sample() per sample, and tests/test_pose_math_host.py compiles this
// same file with g++ and checks it on the CPU against the oracle and the reference fixtures (a test of the SOURCE of
// the device code, not a CPU path of the product: nothing in emoportraits_b200 calls the host build).
//
//   theta  = S.R.T                                   utils/point_transforms.py:187-240
//   mixing = get_mixing_theta                         notebooks/infer.py:686-736 (mix_old False :729, True :727)
//   smooth = exponential smoothing over frames        notebooks/infer.py:571-581
//   warp   = (invert ? inverse(theta) : theta)[:3]    notebooks/infer.py:443 / :586
//   align  = (inverse(theta4)[[0,1,3]][:, [0,1,3]] . diag(.5,.5,1))[:2]   expression_embedder.py:161-203
#pragma once
#include <math.h>

#include "../../include/emoportraits_b200.h"

#if defined(__CUDACC__)
#define EMO_HD __host__ __device__
#else
#define EMO_HD
#endif

namespace emo {
namespace pose {

EMO_HD inline void mat4_mul(const float* a, const float* b, float* c) {
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      float s = 0.f;
      for (int k = 0; k < 4; ++k) s += a[i * 4 + k] * b[k * 4 + j];
      c[i * 4 + j] = s;
    }
}

EMO_HD inline void mat4_mul_d(const double* a, const double* b, double* c) {
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double s = 0.0;
      for (int k = 0; k < 4; ++k) s += a[i * 4 + k] * b[k * 4 + j];
      c[i * 4 + j] = s;
    }
}

// general 4x4 inverse by Gauss-Jordan with partial pivoting, fp32 in/out, fp64 inside
// (torch.inverse is LU in fp32; the fp64 inside only makes us closer to the exact inverse)
EMO_HD inline void mat4_inv(const float* a, float* out) {
  double m[4][8];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) { m[i][j] = a[i * 4 + j]; m[i][4 + j] = (i == j) ? 1.0 : 0.0; }
  for (int c = 0; c < 4; ++c) {
    int piv = c;
    double best = fabs(m[c][c]);
    for (int r = c + 1; r < 4; ++r)
      if (fabs(m[r][c]) > best) { best = fabs(m[r][c]); piv = r; }
    if (piv != c)
      for (int j = 0; j < 8; ++j) { double t = m[c][j]; m[c][j] = m[piv][j]; m[piv][j] = t; }
    const double inv = 1.0 / m[c][c];
    for (int j = 0; j < 8; ++j) m[c][j] *= inv;
    for (int r = 0; r < 4; ++r)
      if (r != c) {
        const double f = m[r][c];
        for (int j = 0; j < 8; ++j) m[r][j] -= f * m[c][j];
      }
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) out[i * 4 + j] = (float)m[i][4 + j];
}

// polar decomposition A = U P of a 3x3 matrix in fp64 (Newton iteration on the orthogonal factor,
// quadratically convergent; scipy.linalg.polar gets the same U, P via SVD)
EMO_HD inline void polar3(const double* A, double* U, double* P) {
  double X[9];
  for (int i = 0; i < 9; ++i) X[i] = A[i];
  for (int it = 0; it < 60; ++it) {
    // inverse transpose of X via cofactors
    double c[9];
    c[0] = X[4] * X[8] - X[5] * X[7]; c[1] = X[5] * X[6] - X[3] * X[8]; c[2] = X[3] * X[7] - X[4] * X[6];
    c[3] = X[2] * X[7] - X[1] * X[8]; c[4] = X[0] * X[8] - X[2] * X[6]; c[5] = X[1] * X[6] - X[0] * X[7];
    c[6] = X[1] * X[5] - X[2] * X[4]; c[7] = X[2] * X[3] - X[0] * X[5]; c[8] = X[0] * X[4] - X[1] * X[3];
    const double det = X[0] * c[0] + X[1] * c[1] + X[2] * c[2];
    double diff = 0.0;
    for (int i = 0; i < 9; ++i) {
      const double nx = 0.5 * (X[i] + c[i] / det);  // c/det = X^{-T}
      diff += fabs(nx - X[i]);
      X[i] = nx;
    }
    if (diff < 1e-15) break;
  }
  for (int i = 0; i < 9; ++i) U[i] = X[i];
  // P = U^T A
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0.0;
      for (int k = 0; k < 3; ++k) s += U[k * 3 + i] * A[k * 3 + j];
      P[i * 3 + j] = s;
    }
  // symmetrise (exact P is symmetric)
  for (int i = 0; i < 3; ++i)
    for (int j = i + 1; j < 3; ++j) { const double s = 0.5 * (P[i * 3 + j] + P[j * 3 + i]); P[i * 3 + j] = s; P[j * 3 + i] = s; }
}

// a*m + b*om with the two products rounded separately, as torch evaluates `x * m + y * (1 - m)` on fp32 tensors
EMO_HD inline float lerp_unfused(float a, float m, float b, float om) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(__fmul_rn(a, m), __fmul_rn(b, om));
#else
  volatile float p = a * m, q = b * om;  // volatile: no contraction into an FMA whatever the host flags
  return p + q;
#endif
}

// S.R.T from (scale xyz, yaw pitch roll, translation xyz); rotation clamped to [-pi/2, pi] (point_transforms.py:197)
EMO_HD inline void theta_from_srt(const float* q, float* th) {
  float S[16] = {q[0], 0, 0, 0, 0, q[1], 0, 0, 0, 0, q[2], 0, 0, 0, 0, 1};
  const float pi = 3.14159265358979323846f;
  const float yaw = fminf(fmaxf(q[3], -pi / 2), pi), pitch = fminf(fmaxf(q[4], -pi / 2), pi), roll = fminf(fmaxf(q[5], -pi / 2), pi);
  // sin/cos evaluated in double and rounded: agrees with the host libm float results the reference gets (cosf/sinf of
  // the CUDA math library may differ from them by 1 ulp, which the 4x4 inverse downstream amplifies)
  const float cy = (float)cos((double)yaw), sy = (float)sin((double)yaw), cp = (float)cos((double)pitch),
              sp = (float)sin((double)pitch), cr = (float)cos((double)roll), sr = (float)sin((double)roll);
  float R[16] = {cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr, 0,
                 sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr, 0,
                 -sp,     cp * sr,                cp * cr,                0,
                 0, 0, 0, 1};
  float T[16] = {1, 0, 0, q[6], 0, 1, 0, q[7], 0, 0, 1, q[8], 0, 0, 0, 1};
  float SR[16];
  mat4_mul(S, R, SR);
  mat4_mul(SR, T, th);
}

// get_mixing_theta for one (source, target) pair, B = T = 1 (notebooks/infer.py:686-736): all on 4x4 float64 matrices
// whose last row/col is that of the identity; the result keeps rows [:3] (the 4th row used downstream is [0,0,0,1],
// expression_embedder.py:163-168).
EMO_HD inline void mix_theta(const float* source_theta, int mix_old, float* th) {
  double As[9], At[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) { As[i * 3 + j] = source_theta[i * 4 + j]; At[i * 3 + j] = th[i * 4 + j]; }
  double Us[9], Ps[9], Ut[9], Pt[9];
  polar3(As, Us, Ps);
  polar3(At, Ut, Pt);
  double Ps4[16] = {0}, Rt[16] = {0}, Tm[16] = {0}, M2[16], M3[16];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) { Ps4[i * 4 + j] = Ps[i * 3 + j]; Rt[i * 4 + j] = Ut[i * 3 + j]; }
  Ps4[15] = 1.0; Rt[15] = 1.0;
  for (int i = 0; i < 4; ++i) Tm[i * 4 + i] = 1.0;
  Tm[3] = th[3]; Tm[7] = th[7]; Tm[11] = th[11];
  if (mix_old) {
    // target_translation @ target_rotation @ source_stretch (:727)
    mat4_mul_d(Tm, Rt, M2);
    mat4_mul_d(M2, Ps4, M3);
  } else {
    // (source_stretch * target_stretch.mean() / source_stretch.mean()) @ target_rotation @ target_translation (:729);
    // .mean() runs over the 4x4 matrices (15 zeros + the trailing 1 included)
    double ms = 1.0, mt = 1.0;
    for (int i = 0; i < 9; ++i) { ms += Ps[i]; mt += Pt[i]; }
    ms /= 16.0; mt /= 16.0;
    const double k = mt / ms;
    double M1[16];
    for (int i = 0; i < 16; ++i) M1[i] = Ps4[i] * k;
    mat4_mul_d(M1, Rt, M2);
    mat4_mul_d(M2, Tm, M3);
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j) th[i * 4 + j] = (float)M3[i * 4 + j];
  th[12] = 0.f; th[13] = 0.f; th[14] = 0.f; th[15] = 1.f;
}

// the whole per-sample pipeline of emo_pose_theta (see include/emoportraits_b200.h)
EMO_HD inline void pose_sample(const emo_pose_desc& d, int n) {
  float th[16];
  if (d.theta_in) {
    for (int i = 0; i < 16; ++i) th[i] = d.theta_in[n * 16 + i];
  } else {
    theta_from_srt(d.srt + n * 9, th);
  }
  if (d.mix) mix_theta(d.source_theta, d.mix_old, th);
  if (d.smooth_state) {
    // self.theta = theta_i * m + self.theta * (1 - m) on rows [:3]; the first frame after a reset seeds the state
    // (notebooks/infer.py:572-577).  Python evaluates 1 - m in double from the unrounded momentum and torch rounds the
    // result to fp32: the caller passes that value, since 1 - fp32(m) rounds differently for momenta like 0.9.  A zero
    // field is a descriptor that predates it (trailing fields zero-initialised): 1 - fp32(m), which is also 0 at m = 1.
    const float m = d.smooth_momentum;
    const float om = d.smooth_one_minus != 0.f ? d.smooth_one_minus : (float)(1.0 - (double)m);
    if (d.smooth_init && n == 0)
      for (int i = 0; i < 12; ++i) d.smooth_state[i] = th[i];
    for (int i = 0; i < 12; ++i) {
      const float v = lerp_unfused(th[i], m, d.smooth_state[i], om);
      d.smooth_state[i] = v;
      th[i] = v;
    }
    th[12] = 0.f; th[13] = 0.f; th[14] = 0.f; th[15] = 1.f;
  }
  if (d.theta_out)
    for (int i = 0; i < 16; ++i) d.theta_out[n * 16 + i] = th[i];
  float inv[16];
  if (d.invert_warp || d.align2d) mat4_inv(th, inv);
  if (d.theta_warp) {
    const float* src = d.invert_warp ? inv : th;
    for (int i = 0; i < 12; ++i) d.theta_warp[n * 12 + i] = src[i];
  }
  if (d.align2d) {
    // inverse()[:, :, [0,1,3]][:, [0,1,3]] then @ diag(0.5, 0.5, 1), rows [:2]
    const int idx[3] = {0, 1, 3};
    for (int i = 0; i < 2; ++i)
      for (int j = 0; j < 3; ++j) {
        const float v = inv[idx[i] * 4 + idx[j]];
        d.align2d[n * 6 + i * 3 + j] = (j < 2) ? v * 0.5f : v;
      }
  }
}

}  // namespace pose
}  // namespace emo
