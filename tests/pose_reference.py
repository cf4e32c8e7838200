"""The pose algebra of emo_pose_theta (emoportraits_b200/csrc/pose_math.cuh) restated in float64, with the error bars the
fp32 kernel is held to, and the host build of the same header.  Shared by tests/test_pose_kernel_gpu.py,
tests/test_op_cases_gpu.py, tests/test_model_op_launches_gpu.py and tests/test_pose_math_host.py.

The restatement starts from the fp32 inputs of one call (exact in float64) and rounds nothing:
  * theta = S.R.T of srt with the rotation clamped to [-pi/2, pi] of the fp32 pi, as the kernel clamps
    (utils/point_transforms.py:187-240), or theta_in;
  * mix: get_mixing_theta (notebooks/infer.py:686-736) through scipy.linalg.polar, in either product form;
  * smoothing: state = theta * m + state * (1 - m) on rows [:3] with the exact momentum (notebooks/infer.py:571-581);
  * warp / align: numpy.linalg.inv of the 4x4 theta (notebooks/infer.py:443, expression_embedder.py:161-203).

Bars, per element of the kernel's fp32 outputs:
  * theta rows 0-2: THETA_REL * max(1, |entry|); row 3 is exactly [0, 0, 0, 1];
  * smoothed theta: the theta bar carried through the recurrence, plus SMOOTH_ROUNDINGS roundings of 2^-24 per step (m and
    1 - m to fp32, the two products, the sum) relative to m |theta| + (1 - m) |state|.  The recurrence multiplies the carried
    error by 1 - m each step, so the bar stays finite for every momentum > 0 and grows by at most one step's term at m = 0;
  * inverse (theta_warp with invert_warp, align2d): INV_C * 2^-24 * cond(theta) * max|inverse| per sample, where cond is
    the 2-norm condition number of the float64 theta.  A smoothed theta carries its smoothing bar into the inverse as a
    relative perturbation of theta: the bar adds cond * max|inverse| * (largest smoothing bar / max|theta|)."""
from __future__ import annotations

import ctypes as C
import pathlib
import subprocess

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
PI32 = float(np.float32(np.pi))      # the kernel's clamp compares against the fp32 pi
THETA_REL = 2e-6
SMOOTH_ROUNDINGS = 3.0
INV_C = 8.0
U = 2.0 ** -24


def srt_theta(srt) -> np.ndarray:
    """(N, 4, 4) float64 S.R.T of (N, 9) (scale xyz, yaw pitch roll, translation xyz)"""
    q = np.asarray(srt, dtype=np.float64).reshape(-1, 9)
    N = q.shape[0]
    yaw, pitch, roll = (np.clip(q[:, 3 + i], -PI32 / 2, PI32) for i in range(3))
    cy, sy, cp, sp, cr, sr = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch), np.cos(roll), np.sin(roll)
    R = np.zeros((N, 4, 4))
    R[:, 0] = np.stack([cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr, 0 * cy], -1)
    R[:, 1] = np.stack([sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr, 0 * cy], -1)
    R[:, 2] = np.stack([-sp, cp * sr, cp * cr, 0 * cy], -1)
    R[:, 3, 3] = 1.0
    S = np.zeros((N, 4, 4))
    S[:, [0, 1, 2], [0, 1, 2]] = q[:, :3]
    S[:, 3, 3] = 1.0
    T = np.tile(np.eye(4), (N, 1, 1))
    T[:, :3, 3] = q[:, 6:9]
    return S @ R @ T


def mix_theta(source_theta, theta, mix_old: bool) -> np.ndarray:
    """get_mixing_theta of each (4, 4) target in `theta` against one (4, 4) source, float64 (last row [0, 0, 0, 1])"""
    from scipy import linalg

    s = np.asarray(source_theta, dtype=np.float64).reshape(4, 4)
    sl = np.eye(4)
    sl[:3, :3] = s[:3, :3]
    _, s_str = linalg.polar(sl)
    out = []
    for t in np.asarray(theta, dtype=np.float64):
        tl, tt = np.eye(4), np.eye(4)
        tl[:3, :3], tt[:3, 3] = t[:3, :3], t[:3, 3]
        t_rot, t_str = linalg.polar(tl)
        out.append(tt @ t_rot @ s_str if mix_old else s_str * t_str.mean() / s_str.mean() @ t_rot @ tt)
    out = np.stack(out)
    out[:, 3] = [0.0, 0.0, 0.0, 1.0]
    return out


def pose64(srt=None, theta_in=None, source_theta=None, mix=False, mix_old=False, momentum=None, init=False, state=None):
    """float64 restatement of one emo_pose_theta call and the bars of its outputs: (ref, bar), dicts of
    theta (N, 4, 4), warp_inv (N, 3, 4), align (N, 2, 3) and, when smoothing (momentum not None), state (3, 4).
    `state` is the (3, 4) state the call starts from (ignored with init).  bar["warp_inv"] and bar["align"] bound the inverse."""
    th = srt_theta(srt) if theta_in is None else np.asarray(theta_in, dtype=np.float64).reshape(-1, 4, 4).copy()
    if mix:
        th = mix_theta(source_theta, th, mix_old)
    N = th.shape[0]
    tbar = THETA_REL * np.maximum(1.0, np.abs(th))
    tbar[:, 3] = 0.0
    ref, bar = {}, {}
    if momentum is not None:
        m = float(momentum)
        s = th[0, :3].copy() if init else np.asarray(state, dtype=np.float64).reshape(3, 4).copy()
        b = tbar[0, :3].copy() if init else np.zeros((3, 4))
        for n in range(N):
            t = th[n, :3]
            new = t * m + s * (1 - m)
            b = m * tbar[n, :3] + (1 - m) * b + SMOOTH_ROUNDINGS * U * (m * np.abs(t) + (1 - m) * np.abs(s))
            s = new
            th[n, :3], tbar[n, :3] = s, b
        ref["state"], bar["state"] = s.copy(), b.copy()
    inv = np.linalg.inv(th)
    cond = np.linalg.cond(th)
    mx = np.abs(inv).reshape(N, -1).max(1)
    smooth_rel = tbar.reshape(N, -1).max(1) / np.abs(th).reshape(N, -1).max(1) if momentum is not None else 0.0
    ibar = (cond * mx * (INV_C * U + smooth_rel))[:, None, None]
    ref["theta"], bar["theta"] = th, tbar
    ref["warp_inv"], bar["warp_inv"] = inv[:, :3], np.broadcast_to(ibar, (N, 3, 4))
    a = inv[:, [0, 1, 3]][:, :, [0, 1, 3]][:, :2] * np.array([0.5, 0.5, 1.0])
    ref["align"], bar["align"] = a, np.broadcast_to(ibar, (N, 2, 3))
    return ref, bar


def excess(got, want, bar) -> float:
    """largest |got - want| / bar (got fp32 torch or numpy; want, bar float64 numpy); where bar is 0 got must equal want"""
    g = np.asarray(got.detach().cpu().numpy() if hasattr(got, "detach") else got, dtype=np.float64)
    d = np.abs(g - want)
    exact = bar == 0
    if exact.any():
        assert (d[exact] == 0).all(), f"{int((d[exact] != 0).sum())} entries that must be exact differ (max {d[exact].max():.2e})"
    return float((d[~exact] / bar[~exact]).max()) if (~exact).any() else 0.0


def _np(x):
    return None if x is None else np.asarray(x.detach().cpu().numpy() if hasattr(x, "detach") else x)


def pose64_of(t: dict, mix="nomix", momentum=None, init=False, state0=None):
    """pose64 of the inputs `t` of one call (srt or theta_in, source_theta; tensors on any device)"""
    return pose64(_np(t.get("srt")), _np(t.get("theta_in")), _np(t.get("source_theta")), mix != "nomix", mix == "mix_old",
                  momentum, init, _np(state0))


def check_outputs(t: dict, o: dict, mix="nomix", invert=False, momentum=None, init=False, state0=None) -> dict:
    """the outputs `o` of one emo_pose_theta call on the inputs `t` against pose64 (see compare); state0: the state a
    carried call started from.  Returns {output: largest error / bar}."""
    return compare(o, *pose64_of(t, mix, momentum, init, state0), invert)


def compare(o: dict, ref: dict, bar: dict, invert: bool) -> dict:
    """the outputs `o` (theta_out, theta_warp and, if set, align2d and smooth_state) against pose64's (ref, bar): every
    element written, every entry within its bar, theta_out row 3 exactly [0, 0, 0, 1].  Returns {output: largest error / bar}."""
    for name, v in o.items():
        assert not np.isnan(_np(v)).any(), f"{name}: {int(np.isnan(_np(v)).sum())} elements never written"
    th = _np(o["theta_out"])
    assert (th[:, 3] == np.array([0, 0, 0, 1], np.float32)).all(), "theta_out row 3 is not [0, 0, 0, 1]"
    e = {"theta_out": excess(th, ref["theta"], bar["theta"])}
    e["theta_warp"] = (excess(o["theta_warp"], ref["warp_inv"], bar["warp_inv"]) if invert
                       else excess(o["theta_warp"], ref["theta"][:, :3], bar["theta"][:, :3]))
    if o.get("align2d") is not None:
        e["align2d"] = excess(o["align2d"], ref["align"], bar["align"])
    if o.get("smooth_state") is not None:
        e["smooth_state"] = excess(o["smooth_state"], ref["state"], bar["state"])
    for name, v in e.items():
        assert v <= 1.0, f"{name}: error {v:.2f} x its float64 bar"
    return e


# ------------------------------------------------------------------------------------------------------------------
# the host build of pose_math.cuh
# ------------------------------------------------------------------------------------------------------------------
SHIM = r'''
#include "emoportraits_b200/csrc/pose_math.cuh"
extern "C" void pose_host(const emo_pose_desc* d) {
  for (int n = 0; n < d->N; ++n) emo::pose::pose_sample(*d, n);
}
'''


def host_build(tmp: pathlib.Path):
    """compile the header for the CPU (g++, no FMA contraction) and return run(**kw) -> (theta, warp, align) as torch
    tensors.  run takes the arguments of ops.pose_theta as numpy-convertible arrays; smooth_state (a float32 numpy array) is
    updated in place."""
    import torch

    from emoportraits_b200 import ops

    (tmp / "shim.cpp").write_text(SHIM)
    so = tmp / "libpose_host.so"
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-I", str(ROOT), "-x", "c++",
                    str(tmp / "shim.cpp"), "-o", str(so)], check=True)
    lib = C.CDLL(str(so))
    lib.pose_host.argtypes = [C.c_void_p]
    lib.pose_host.restype = None

    def run(srt=None, source_theta=None, mix=False, invert_warp=False, mix_old=False, theta_in=None, smooth_state=None,
            smooth_momentum=0.5, smooth_init=False):
        ref = srt if srt is not None else theta_in
        N = ref.shape[0]
        f = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float32)  # noqa: E731
        srt, source_theta, theta_in = f(srt), f(source_theta), f(theta_in)
        if smooth_state is not None:
            assert smooth_state.dtype == np.float32 and smooth_state.flags.c_contiguous
        theta, warp, align = (np.zeros((N, 4, 4), np.float32), np.zeros((N, 3, 4), np.float32), np.zeros((N, 2, 3), np.float32))
        p = lambda a: None if a is None else a.ctypes.data  # noqa: E731
        d = ops.pose_desc(N, p(srt), p(source_theta), p(theta), p(warp), p(align), p(theta_in), p(smooth_state), mix=mix,
                          invert_warp=invert_warp, mix_old=mix_old, smooth_init=smooth_init, smooth_momentum=smooth_momentum)
        lib.pose_host(C.byref(d))
        return torch.from_numpy(theta), torch.from_numpy(warp), torch.from_numpy(align)

    return run
