"""GPU tests of the device pose kernel (emo_pose_theta, pose_theta_kernel in emoportraits_b200/csrc/misc.cu, whose body is
csrc/pose_math.cuh) on every emo_pose_theta case of tests/op_cases.py: srt or a sheared theta_in, no mix / mix / mix_old,
invert_warp on and off, align2d set and NULL, N of 1, 32, 33 and 300, angles inside the [-pi/2, pi] clamp, beyond it and on
its edges, and smoothing at eight momenta.

A smoothing case that carries its state runs as two calls: one that seeds the state (smooth_init) on the case's first three
samples, then the case's call on all its samples from that state.  Per case:
  * every output within its float64 bar (tests/pose_reference.py), the two calls restated as one sequence;
  * theta_out row 3 exactly [0, 0, 0, 1];
  * smoothing: the smoothed theta_out, the non-inverted theta_warp and the final smooth_state equal, bit for bit, the
    reference's own fp32 recurrence `theta * m + state * (1 - m)` (notebooks/infer.py:577) run by torch on the CPU over
    the kernel's unsmoothed theta_out of the same calls;
  * the host build of pose_math.cuh (g++, no contraction) within the same bars, and bit for bit equal where the device
    cannot contract either (theta_in, no mix, no inverse: theta_out and theta_warp, smoothed or not);
  * every output element written, the NaN guard after each output and after the 12 floats of smooth_state untouched;
  * two runs bit-identical.
The report prints the largest error as a fraction of its bar per class, and the largest device-to-host difference per output."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import op_cases as OC
import pose_reference as PR

pytestmark = pytest.mark.gpu
GUARD = 64
POSE = [c for c in OC.CASES if c.op == "pose_theta"]
PRE = 3            # samples of the call that seeds the state before a carried case
_WORST, _HOST = {}, {}


@pytest.fixture(scope="module")
def ops():
    from emoportraits_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return PR.host_build(tmp_path_factory.mktemp("pose_host"))


def _calls(c, t):
    """[(inputs, smooth_init)] of the case: the seeding call first for a carried smoothing case"""
    k = c.k
    if "smooth" not in k or k["init"]:
        return [(t, k.get("init", False))]
    first = {n: (v[:PRE].contiguous() if n in ("srt", "theta_in") else v) for n, v in t.items() if n != "state0"}
    return [(first, True), ({n: v for n, v in t.items() if n != "state0"}, False)]


def _device(ops, c, calls, smooth=True):
    """run `calls` on the device with guarded NaN outputs; returns the outputs of every call concatenated (CPU), the final
    state, and checks that every element is written and no guard changed"""
    from emoportraits_b200 import lib as L

    k = c.k
    sm = "smooth" in k and smooth
    sbuf = torch.full((12 + GUARD,), float("nan"), device="cuda") if sm else None
    outs = []
    for ti, init in calls:
        N = (ti.get("srt") if "srt" in ti else ti["theta_in"]).shape[0]
        shapes = {"theta_out": (N, 4, 4), "theta_warp": (N, 3, 4)}
        if k["align"]:
            shapes["align2d"] = (N, 2, 3)
        bufs = {n: torch.full((math.prod(s) + GUARD,), float("nan"), device="cuda") for n, s in shapes.items()}
        o = {n: bufs[n][:math.prod(s)].view(s) for n, s in shapes.items()}
        p = ops._p
        d = ops.pose_desc(N, p(ti.get("srt")), p(ti.get("source_theta")), p(o["theta_out"]), p(o["theta_warp"]), p(o.get("align2d")),
                          p(ti.get("theta_in")), p(sbuf) if sm else None, mix=k["mix"] != "nomix", invert_warp=k["invert"],
                          mix_old=k["mix"] == "mix_old", smooth_init=init, smooth_momentum=k.get("smooth", 0.5))
        L.call("emo_pose_theta", C.byref(d), ops._stream())
        torch.cuda.synchronize()
        for n, s in shapes.items():
            assert torch.isnan(bufs[n][math.prod(s):]).all(), f"{n}: write past the end"
            assert not torch.isnan(o[n]).any(), f"{n}: {int(torch.isnan(o[n]).sum())} elements never written"
        outs.append({n: v.cpu() for n, v in o.items()})
    out = {n: torch.cat([x[n] for x in outs]) for n in outs[0]}
    if sm:
        assert torch.isnan(sbuf[12:]).all(), "smooth_state: write past its 12 floats"
        assert not torch.isnan(sbuf[:12]).any(), "smooth_state not written"
        out["smooth_state"] = sbuf[:12].view(3, 4).cpu()
    return out


def _host(host, c, calls):
    """the same calls through the host build"""
    k = c.k
    state = np.full((3, 4), np.nan, np.float32) if "smooth" in k else None
    outs = []
    for ti, init in calls:
        n = lambda x: None if x is None else x.cpu().numpy()  # noqa: E731
        th, wp, al = host(srt=n(ti.get("srt")), theta_in=n(ti.get("theta_in")), source_theta=n(ti.get("source_theta")),
                          mix=k["mix"] != "nomix", mix_old=k["mix"] == "mix_old", invert_warp=k["invert"], smooth_state=state,
                          smooth_momentum=k.get("smooth", 0.5), smooth_init=init)
        outs.append(dict(theta_out=th, theta_warp=wp, **({"align2d": al} if k["align"] else {})))
    out = {n: torch.cat([x[n] for x in outs]) for n in outs[0]}
    if state is not None:
        out["smooth_state"] = torch.from_numpy(state)
    return out


def _sequence(calls):
    """the inputs of the calls as one sequence of samples (the state carries from one call to the next)"""
    t = dict(calls[0][0])
    for n in ("srt", "theta_in"):
        if n in t:
            t[n] = torch.cat([ti[n] for ti, _ in calls])
    return t


def _note(table, key, v, cid):
    if v > table.get(key, (-1.0, ""))[0]:
        table[key] = (v, cid)


@pytest.mark.parametrize("c", POSE, ids=[c.id for c in POSE])
def test_pose_kernel_case(ops, host, c):
    k = c.k
    t = OC.inputs(c, "cuda")
    calls = _calls(c, t)
    got = _device(ops, c, calls)
    again = _device(ops, c, calls)
    for n in got:
        assert torch.equal(got[n].view(torch.int32), again[n].view(torch.int32)), f"{n}: two runs differ"

    seq = _sequence(calls)
    e = PR.check_outputs(seq, got, k["mix"], k["invert"], k.get("smooth"), calls[0][1], None)
    _note(_WORST, c.want, max(e.values()), c.id)

    # the host build: within the same bars, bit for bit where nothing can be contracted
    hb = _host(host, c, calls)
    eh = PR.check_outputs(seq, hb, k["mix"], k["invert"], k.get("smooth"), calls[0][1], None)
    _, bar = PR.pose64(*(None if seq.get(n) is None else seq[n].cpu().numpy() for n in ("srt", "theta_in", "source_theta")),
                         k["mix"] != "nomix", k["mix"] == "mix_old", k.get("smooth"), calls[0][1], None)
    bars = {"theta_out": bar["theta"], "theta_warp": bar["warp_inv"] if k["invert"] else bar["theta"][:, :3],
            "align2d": bar["align"], "smooth_state": bar.get("state")}
    exact = k["src"] == "theta_in" and k["mix"] == "nomix" and not k["invert"]
    msg = f"\n[{c.id}] {c.want}: error / bar " + " ".join(f"{n} {v:.2f}" for n, v in e.items()) + "; device - host"
    for n in got:
        d = (got[n].double() - hb[n].double()).abs()
        b = torch.from_numpy(np.ascontiguousarray(bars[n]))
        assert (d <= b).all(), f"{n}: device and host builds differ by {d.max().item():.2e}, beyond the float64 bar"
        if exact and n in ("theta_out", "theta_warp"):
            assert torch.equal(got[n], hb[n]), f"{n}: device and host builds differ where neither can contract"
        _note(_HOST, n, d.max().item(), c.id)
        msg += f" {n} {d.max().item():.1e}"
    print(msg + (" (host build within its bars: " + " ".join(f"{n} {v:.2f}" for n, v in eh.items()) + ")"))


@pytest.mark.parametrize("c", [c for c in POSE if "smooth" in c.k], ids=[c.id for c in POSE if "smooth" in c.k])
def test_smoothing_is_the_reference_fp32_recurrence(ops, c):
    """the smoothed outputs are the reference's fp32 recurrence over the kernel's own unsmoothed poses, bit for bit: the
    state is multiplied by fp32(1 - m) with 1 - m taken in double, which 1 - fp32(m) is not for momenta like 0.9"""
    from oracle import restatement as R

    k = c.k
    calls = _calls(c, OC.inputs(c, "cuda"))
    got = _device(ops, c, calls)
    plain = _device(ops, c, calls, smooth=False)["theta_out"]
    state = {"theta": None}
    want = R.smooth_theta(state, plain[:, :3], k["smooth"])
    assert torch.equal(got["theta_out"][:, :3], want), (got["theta_out"][:, :3] - want).abs().max().item()
    assert torch.equal(got["smooth_state"], state["theta"]), (got["smooth_state"] - state["theta"]).abs().max().item()
    if not k["invert"]:
        assert torch.equal(got["theta_warp"], want)


def test_report_pose_kernel():
    """(runs after the cases) the largest error / float64 bar per class, and the largest device-to-host difference per
    output"""
    if not _WORST:
        pytest.skip("no pose case ran")
    for cls, (v, cid) in sorted(_WORST.items()):
        print(f"\n[largest error / bar] {cls:36s} {v:.3f}  ({cid})", end="")
    for n, (v, cid) in sorted(_HOST.items()):
        print(f"\n[largest |device - host build|] {n:14s} {v:.2e}  ({cid})", end="")
