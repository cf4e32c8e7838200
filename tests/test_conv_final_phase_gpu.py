"""Every instantiation of the convolution kernel's final phase against float64.

The in-kernel final phase (bias, residual, activation, post-add, stores, GroupNorm statistics) is compiled once per
activation for even channel counts (float2 stores) and once more for odd channel counts (scalar path, activation read at
run time).  These cases run each of them, in channels-last and NCHW output, on the kernel forms the models use, with the
K loop in one CTA (no split-K finalize).  Same bar as tests/test_conv_plan_gpu.py: within 2e-5 of the scale, statistics
against the float64 group means, every output element written (it starts as NaN) and nothing written past the output (a
NaN guard follows it)."""
import math

import pytest
import torch

import conv_plan_cases as CP

pytestmark = pytest.mark.gpu
GUARD = 4096
TOL = 2e-5
ACTS = [0, CP.RELU, CP.SIGMOID, CP.TANH]


def _cases():
    cases = []
    for act in ACTS:
        # even channel counts: the float2 path of this activation
        cases += [
            CP.Case("", 64, 96, (192, 160), planes=CP.B2, split_k=False, residual=True, post_add=True, stats=True, act=act),
            CP.Case("", 128, 80, (96, 96), planes=CP.B2, split_k=False, residual=True, res_shift=1, stats=True, G=16, act=act),
            CP.Case("", 64, 64, (80, 72), planes=CP.B2, split_k=False, out_nchw=True, post_add=True, act=act, N=2),
            CP.Case("", 64, 48, (8, 32, 48), planes=CP.H2, split_k=False, residual=True, stats=True, G=8, act=act),
            CP.Case("", 96, 112, (96, 96), planes=CP.B3, split_k=False, post_add=True, act=act),
            CP.Case("", 64, 64, (48, 48), upconv=True, split_k=False, post_add=True, stats=True, act=act),
            # odd channel counts: the scalar path
            CP.Case("", 64, 3, (96, 96), planes=CP.B2, split_k=False, residual=True, post_add=True, act=act),
            CP.Case("", 32, 7, (64, 72), planes=CP.B3, split_k=False, out_nchw=True, act=act, N=2),
        ]
    return cases


CASES = _cases()


@pytest.fixture(scope="module")
def ops():
    from emoportraits_b200 import ops as o
    return o


def _to_ncdhw(c, t):
    t = t if c.out_nchw else t.permute(0, 4, 1, 2, 3)
    return t if len(c.sp) == 3 else t[:, :, 0]


@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_final_phase_against_float64(ops, c):
    from emoportraits_b200 import lib as L

    x, w, b, res, pa = CP.make(c, "cuda")
    Do, Ho, Wo = CP.out_shape(c)
    shape = (c.N, c.Cout, Do, Ho, Wo) if c.out_nchw else (c.N, Do, Ho, Wo, c.Cout)
    numel = math.prod(shape)
    buf = torch.full((numel + GUARD,), float("nan"), device="cuda")
    out = buf[:numel].view(shape)
    st = torch.zeros((c.N, c.G, 2), dtype=torch.float64, device="cuda") if c.stats else None
    a, pw, kw = CP.conv_args(c, ops, x, w, b, res, pa, stats=st, out=out)
    info = ops.conv_plan(a, pw, **kw)
    assert info.ksplit == 1 and L.CONV_FINISH[info.finish] == "none", CP.plan_class(info, CP.depth(c))

    ops.conv_igemm(a, pw, **kw)
    torch.cuda.synchronize()
    ref, scale = CP.reference(c, x, w, b, res, pa)
    assert torch.isnan(buf[numel:]).all(), "write past the end of the output tensor"
    assert not torch.isnan(out).any(), f"{int(torch.isnan(out).sum())} output elements never written"
    e = (_to_ncdhw(c, out).double() - ref).abs().max().item()
    assert e < TOL * max(1.0, scale), (CP.plan_class(info, CP.depth(c)), e, scale)
    if st is not None:
        r = ref.reshape(c.N, c.G, -1)
        count = r.shape[-1]
        d_mean = ((st[..., 0] / count - r.mean(-1)).abs()).max().item()
        msq = (r * r).mean(-1)
        d_msq = ((st[..., 1] / count - msq).abs() / msq).max().item()
        assert d_mean < 1e-6 * max(1.0, scale) and d_msq < 1e-5, (d_mean, d_msq)
    print(f"\n[{c.id}] {CP.plan_class(info, CP.depth(c))}: max-abs {e:.2e} (scale {scale:.2f})")
