"""CPU test of the SOURCE of the device pose algebra.  emoportraits_b200/csrc/pose_math.cuh is host+device code: the
CUDA kernel pose_theta_kernel calls pose::pose_sample() per sample; here the same file is compiled with g++ and driven
through the same emo_pose_desc (ctypes structure of emoportraits_b200/lib.py) with HOST pointers, and compared with
the oracle (oracle/restatement.py: torch + scipy.linalg.polar, as the reference computes it) and with the poses the
unmodified reference produced (tests/golden/va256_options.pt).  The build itself is tests/pose_reference.host_build, which
tests/test_pose_kernel_gpu.py compares the device build with.  This is test infrastructure: the product never calls
the host build (the GPU parity tests call the kernel through the C-ABI)."""
import pathlib

import numpy as np
import pytest
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
GOLD = ROOT / "tests" / "golden"


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    import pose_reference as PR

    return PR.host_build(tmp_path_factory.mktemp("pose_host"))


def _srt(n, seed, wild=False):
    g = torch.Generator().manual_seed(seed)
    s = 1 + 0.2 * (torch.rand(n, 3, generator=g) - 0.5)
    r = (torch.rand(n, 3, generator=g) - 0.5) * (8.0 if wild else 1.2)   # wild: beyond the [-pi/2, pi] clamp
    t = (torch.rand(n, 3, generator=g) - 0.5) * 0.3
    return torch.cat([s, r, t], 1)


@pytest.mark.parametrize("wild", [False, True])
def test_theta_inverse_and_alignment(host, wild):
    from oracle import restatement as R

    srt = _srt(64, 3, wild)
    ref = R.get_transform_matrix(srt[:, :3], srt[:, 3:6], srt[:, 6:9])
    theta, warp, align = host(srt.numpy(), invert_warp=True)
    assert (theta - ref).abs().max().item() < 2e-6
    assert (warp - ref.inverse()[:, :3]).abs().max().item() < 2e-5
    assert (align - R.align_theta_2d(ref[:, :3])).abs().max().item() < 2e-5
    _, warp_fwd, _ = host(srt.numpy(), invert_warp=False)
    assert torch.equal(warp_fwd, theta[:, :3])


@pytest.mark.parametrize("mix_old", [False, True])
def test_mixing_matches_scipy_polar(host, mix_old):
    from oracle import restatement as R

    src = _srt(1, 7)
    ths = R.get_transform_matrix(src[:, :3], src[:, 3:6], src[:, 6:9])
    srt = _srt(32, 8)
    thd = R.get_transform_matrix(srt[:, :3], srt[:, 3:6], srt[:, 6:9])
    ref = torch.cat([R.get_mixing_theta(ths, thd[i:i + 1], mix_old) for i in range(srt.shape[0])])
    theta, warp, align = host(srt.numpy(), source_theta=ths[0].numpy(), mix=True, mix_old=mix_old)
    assert (theta[:, :3] - ref).abs().max().item() < 1e-6
    assert torch.equal(theta[:, 3], torch.tensor([0., 0., 0., 1.]).expand(32, 4))
    assert (align - R.align_theta_2d(ref)).abs().max().item() < 2e-5
    # theta_in replaces S.R.T: same result when fed the matrices themselves
    theta2, _, _ = host(theta_in=thd.numpy(), source_theta=ths[0].numpy(), mix=True, mix_old=mix_old)
    assert (theta2 - theta).abs().max().item() < 1e-6


@pytest.mark.parametrize("momentum", [0.5, 0.3, 0.9, 0.6, 0.99])
def test_smoothing_is_the_reference_recurrence_bit_for_bit(host, momentum):
    from oracle import restatement as R

    srt = _srt(5, 11)
    th = R.get_transform_matrix(srt[:, :3], srt[:, 3:6], srt[:, 6:9])
    state_ref = {"theta": None}
    ref = torch.cat([R.smooth_theta(state_ref, th[:3, :3], momentum), R.smooth_theta(state_ref, th[3:, :3], momentum)])
    state = np.zeros((3, 4), np.float32)
    a, _, _ = host(theta_in=th[:3].numpy(), smooth_state=state, smooth_momentum=momentum, smooth_init=True)
    b, wb, _ = host(theta_in=th[3:].numpy(), smooth_state=state, smooth_momentum=momentum)      # state carried across calls
    got = torch.cat([a, b])[:, :3]
    assert torch.equal(got, ref), (got - ref).abs().max()
    assert torch.equal(torch.from_numpy(state), ref[-1])
    assert torch.equal(wb, b[:, :3])


def test_reference_fixture_poses(host):
    """poses of the UNMODIFIED reference (tests/golden/va256_options.pt) from the regressor output the oracle computes"""
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict
    from oracle import frames as FR
    from oracle import restatement as R
    from oracle.make_golden import option_inputs
    from emoportraits_b200.config import shipped_config

    gold = torch.load(GOLD / "va256_options.pt", weights_only=False)
    hsd = synthetic_head_pose_state_dict(0)
    cases = gold["cases"]
    with torch.no_grad():
        srt_s = R.head_pose(hsd, FR.frame(256, gold["src_seed"], gold["kind"]))
        srt_d = [R.head_pose(hsd, FR.frame(256, s, gold["kind"])) for s in gold["drv_seeds"]]
    ths, _, _ = host(srt_s.numpy())
    src = ths[0].numpy()
    tol = 2e-6
    th, _, _ = host(srt_d[0].numpy(), source_theta=src, mix=True)
    assert (th[:, :3] - cases["default"]["pred_target_theta"][:, :3]).abs().max().item() < tol
    th, _, _ = host(srt_d[0].numpy(), source_theta=src, mix=True, mix_old=True)
    assert (th[:, :3] - cases["mix_old"]["pred_target_theta"][:, :3]).abs().max().item() < tol
    th, _, _ = host(srt_d[0].numpy())
    assert (th[:, :3] - cases["no_mix"]["pred_target_theta"][:, :3]).abs().max().item() < tol
    state = np.zeros((3, 4), np.float32)
    for i, q in enumerate(srt_d):
        th, _, _ = host(q.numpy(), source_theta=src, mix=True, smooth_state=state, smooth_momentum=0.5, smooth_init=(i == 0))
        assert (th[:, :3] - cases[f"smooth_pose_{i}"]["pred_target_theta"][:, :3]).abs().max().item() < tol, i
    X = option_inputs(256, shipped_config(256))
    th, _, _ = host(torch.cat(X["theta_embed"], 1).numpy(), source_theta=src, mix=True)
    assert (th[:, :3] - cases["custome_target_theta_embed"]["pred_target_theta"][:, :3]).abs().max().item() < tol
