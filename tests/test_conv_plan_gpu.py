"""GPU sweep of the implicit-GEMM convolution: every case of tests/conv_plan_cases.py (one per launch configuration the
planner can pick, see tests/test_conv_plan_cpu.py) against float64, plus the accumulation-bias check of the chunked
tensor-core accumulation.

Per case: the plan at the live device's SM count is the class the case names (checked on 132-SM devices only; other SM
counts plan differently); the output matches float64 within 2e-5 of its scale (the largest value accumulated or added);
the GroupNorm statistics give the
float64 per-group mean and mean square; every element of the output tensor is written (it starts as NaN) and nothing is
written past it (a NaN guard region follows it in the same allocation)."""
import math

import pytest
import torch

import conv_plan_cases as CP

pytestmark = pytest.mark.gpu
GUARD = 4096  # floats of NaN after the output tensor
TOL = 2e-5    # max-abs error / max(1, scale), the bar of tests/test_ops_gpu.py
_WORST = {}   # kernel instantiation -> (largest error / max(1, scale), case id)


@pytest.fixture(scope="module")
def ops():
    from emoportraits_b200 import ops as o
    return o


def _to_ncdhw(c, t):
    """a channels-last (N, D, H, W, C) or NCDHW output -> the reference's NCHW / NCDHW layout"""
    t = t if c.out_nchw else t.permute(0, 4, 1, 2, 3)
    return t if len(c.sp) == 3 else t[:, :, 0]


@pytest.mark.parametrize("c", CP.CASES, ids=[c.id for c in CP.CASES])
def test_conv_case_against_float64(ops, c):
    from emoportraits_b200 import lib as L

    x, w, b, res, pa = CP.make(c, "cuda")
    Do, Ho, Wo = CP.out_shape(c)
    shape = (c.N, c.Cout, Do, Ho, Wo) if c.out_nchw else (c.N, Do, Ho, Wo, c.Cout)
    numel = math.prod(shape)
    buf = torch.full((numel + GUARD,), float("nan"), device="cuda")
    out = buf[:numel].view(shape)
    st = torch.zeros((c.N, c.G, 2), dtype=torch.float64, device="cuda") if (c.stats or c.post) else None
    a, pw, kw = CP.conv_args(c, ops, x, w, b, res, pa, stats=st, out=out)

    info = ops.conv_plan(a, pw, **kw)
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    if sms == CP.SM_COUNT:
        assert CP.plan_class(info, CP.depth(c)) == c.want, (CP.plan_class(info, CP.depth(c)), c.want)
    else:
        print(f"\n[{c.id}] {sms} SMs, not {CP.SM_COUNT}: plan class {CP.plan_class(info, CP.depth(c))} not checked against "
              f"{c.want}")
    finish = L.CONV_FINISH[info.finish]

    got = ops.conv_igemm(a, pw, **kw)
    torch.cuda.synchronize()
    ref, scale = CP.reference(c, x, w, b, res, pa)
    assert torch.isnan(buf[numel:]).all(), "write past the end of the output tensor"
    kern = L.CONV_KERNELS[info.kernel]
    msg = f"\n[{c.id}] {CP.plan_class(info, CP.depth(c))} ksplit {info.ksplit} grid {info.grid}:"
    if finish != "post":      # the fused split-K post kernel writes the post-op's output only
        assert not torch.isnan(out).any(), f"{int(torch.isnan(out).sum())} output elements never written"
        err = (_to_ncdhw(c, out).double() - ref).abs()
        e = err.max().item()
        worst = err.flatten(2).amax(-1)   # (N, C): where the error sits if the bound is missed
        msg += f" max-abs {e:.2e} (scale {scale:.2f})"
        rel = e / max(1.0, scale)
        if rel > _WORST.get(kern, (0.0, ""))[0]:
            _WORST[kern] = (rel, c.id)
        assert e < TOL * max(1.0, scale), (e, scale, "worst channels", worst.argmax(-1).tolist())
    if c.post:
        pref = CP.post_reference(c, ref, c.G)
        pe = (_to_ncdhw(c, got).double() - pref).abs().max().item()
        msg += f" post-op max-abs {pe:.2e}"
        assert pe < 5e-5 * max(1.0, pref.abs().max().item()), pe
    if st is not None:
        # statistics in the terms GroupNorm consumes them: per-group mean and mean square
        r = ref.reshape(c.N, c.G, -1)
        count = r.shape[-1]
        d_mean = ((st[..., 0] / count - r.mean(-1)).abs()).max().item()
        msq = (r * r).mean(-1)
        d_msq = ((st[..., 1] / count - msq).abs() / msq).max().item()
        msg += f" stats: mean {d_mean:.1e} mean-square {d_msq:.1e} (rel)"
        assert d_mean < 1e-6 * max(1.0, scale) and d_msq < 1e-5, (d_mean, d_msq)
    print(msg)


# ------------------------------------------------------------------------------------------------------------------
# accumulation bias: the tensor core accumulates with truncation, so the kernel adds short wgmma chunks into fp32 registers
# (emo_conv_desc.acc_chunk_mmas, tools/accum_probe.py).  With non-negative operands the truncation errors all have one
# sign: their mean is the bias.  One accumulation chain over the whole K loop (acc_chunk_mmas = 1 << 20) is the negative
# control: the check must see its bias.
# ------------------------------------------------------------------------------------------------------------------
# H100 SXM (132 SMs, 400 W power limit), first run: default chunks -1.8e-6 / -1.9e-6 (bf16 planes, 1x1 x 1536 / 3x3 x 512:
# 3 / 9 chunks of 96 MMAs), -7.0e-7 / -7.2e-7 (fp16 planes, 12 / 36 chunks of 24); one chain -6.9e-6 / -2.6e-5 (bf16), -1.2e-5 / -3.8e-5 (fp16)
BIAS_BOUND = 3e-6          # |mean signed error| / mean |ref| with the default chunks
CONTROL_FACTOR = 3.0       # the single chain's bias is at least this many times larger, and out of BIAS_BOUND


@pytest.mark.parametrize("planes", [2, "h2"])
@pytest.mark.parametrize("Cin,k", [(1536, 1), (512, 3)])
def test_accumulation_bias_against_float64(ops, Cin, k, planes):
    c = CP.Case("", Cin, 128, (32, 32), k=k, planes=planes, split_k=False, bias=False)
    x, w, _, _, _ = CP.make(c, "cuda", positive=True)
    ref, _ = CP.reference(c, x, w, None, None, None)

    def bias(acc):
        a, pw, kw = CP.conv_args(c, ops, x, w, None, None, None, acc=acc)
        out = ops.conv_igemm(a, pw, **kw)
        torch.cuda.synchronize()
        return ((_to_ncdhw(c, out).double() - ref).mean() / ref.abs().mean()).item()

    b_def, b_one = bias(0), bias(1 << 20)
    print(f"\n[accumulation bias {Cin} ch k{k} planes {planes}] default chunks {b_def:+.2e}, one chain {b_one:+.2e} (relative to mean |ref|)")
    assert abs(b_def) < BIAS_BOUND, b_def
    assert b_one < -BIAS_BOUND and abs(b_one) > CONTROL_FACTOR * abs(b_def), (b_def, b_one)   # truncation: negative


def test_report_largest_error_per_kernel():
    """(runs after the sweep) the largest error / max(1, scale) seen per kernel instantiation"""
    if not _WORST:
        pytest.skip("no sweep case ran")
    for k, (rel, cid) in sorted(_WORST.items()):
        print(f"\n[largest relative error] {k:12s} {rel:.2e}  ({cid})", end="")
