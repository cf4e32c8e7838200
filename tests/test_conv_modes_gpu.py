"""GPU parity of the convolution modes beyond the plain two/three-plane implicit GEMM (tests/test_ops_gpu.py):
  * sub-pixel form of `nearest x2 -> 3x3 conv` (emo_conv_desc.upconv; weight folding checked on the CPU by tests/test_upconv_fold.py),
  * `3x3 conv -> 2x2 avgpool` folded into one 4x4 stride-2 convolution (ops.fold_poolconv_weight),
  * fp16 two-plane operands ("h2": fp32-faithful at three MMAs per product),
each at op level against torch fp64 / the plain kernel, and at model level against the reference fixtures."""
import pathlib

import pytest
import torch

from oracle import frames as FR

pytestmark = pytest.mark.gpu
GOLD = pathlib.Path(__file__).parent / "golden"
SIZE = 256
IMG_TOL = 1e-3      # BASELINE.json north_star: max-abs per pixel on the fp32 image
THETA_TOL = 1e-5


def _img_err(got, ref):
    vals, stride = ref
    return (got.detach().float().cpu().reshape(-1)[::stride] - vals).abs().max().item()


@pytest.fixture(scope="module")
def ctx():
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import Model
    from oracle.make_golden import option_inputs

    cfg = shipped_config(SIZE)
    sd, hsd = synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0)
    model = Model(cfg, sd, hsd, "cuda")
    gold = torch.load(GOLD / f"va{SIZE}_options.pt", weights_only=False)
    src = FR.frame(SIZE, gold["src_seed"], gold["kind"]).cuda()
    drv = [FR.frame(SIZE, s, gold["kind"]).cuda() for s in gold["drv_seeds"]]
    return dict(cfg=cfg, sd=sd, hsd=hsd, model=model, gold=gold["cases"], src=src, drv=drv, X=option_inputs(SIZE, cfg),
                st=model.source_pass(src))


def _check(case, img, so, name):
    e_img = _img_err(img, case["img"])
    e_th = (so.pred_target_theta[:, :3].cpu() - case["pred_target_theta"][:, :3]).abs().max().item()
    e_pe = (so.target_pose_embed.cpu() - case["target_pose_embed"]).abs().max().item()
    print(f"\n[options parity vs reference @256] {name}: img {e_img:.2e} theta {e_th:.2e} pose_embed {e_pe:.2e}")
    assert e_th < THETA_TOL, (name, e_th)
    assert e_pe < 1e-4, (name, e_pe)
    assert e_img < IMG_TOL, (name, e_img)


# ------------------------------------------------------------------------------------------------------------------
# sub-pixel up-sampling convolution (emo_conv_desc.upconv).  The weight folding and the kernel's index arithmetic are
# checked on the CPU by tests/test_upconv_fold.py.
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Cin,Cout,S,residual", [(192, 128, 64, False), (320, 192, 32, True), (512, 320, 32, False),
                                                 (192, 128, 256, True)])
def test_upconv_subpixel_matches_conv_on_upsampled_planes(Cin, Cout, S, residual):
    """conv_igemm(low-res planes, folded weights, upconv=True) == conv_igemm(nearest-x2 planes, 3x3 weights): same operands
    up to the fp32 pre-summing of the folded taps, so agreement to ~2^-15 of the output scale; statistics likewise.
    At 132 SMs the cases plan ps<64,2> with BN 128 (row reuse, 2 halo tiles; S = 256 gives 4096 work items), BN 32 and BN 80
    (3 halo tiles); tests/test_conv_plan_gpu.py sweeps every plan class of this kernel."""
    import math

    from emoportraits_b200 import ops

    g = torch.Generator().manual_seed(Cin + S)
    x = torch.randn((1, 1, S, S, Cin), generator=g).cuda()
    w = torch.randn((Cout, Cin, 3, 3), generator=g) / math.sqrt(9 * Cin)
    b = torch.randn(Cout, generator=g).cuda()
    res = torch.randn((1, 1, S, S, Cout), generator=g).cuda() if residual else None   # low-res skip, read with res_shift = 1
    ops.begin_pass("cuda")                      # zeroed statistics arena for new_stats()
    a_lo = ops.apply(x, act=ops.ACT_RELU, up=1)
    a_up = ops.apply(x, act=ops.ACT_RELU, up=2)
    st_ref, st_ps = ops.new_stats(1, 32, "cuda"), ops.new_stats(1, 32, "cuda")
    ref = ops.conv_igemm(a_up, ops.pack_conv_weight(w), bias=b, residual=res, res_shift=1 if residual else 0, stats=st_ref)
    out = ops.conv_igemm(a_lo, ops.pack_upconv_weight(w), bias=b, residual=res, res_shift=1 if residual else 0, stats=st_ps,
                         upconv=True)
    torch.cuda.synchronize()
    assert out.shape == ref.shape == (1, 1, 2 * S, 2 * S, Cout)
    scale = ref.abs().max().item()
    err = (out - ref).abs().max().item()
    print(f"\n[upconv sub-pixel vs upsampled planes] {Cin}->{Cout} @{S}^2: max-abs {err:.2e} (scale {scale:.2f})")
    assert err < scale * 2 ** -13
    # statistics, in the terms GroupNorm consumes them: per-group mean and mean square.  (The raw sums of the two kernels
    # differ by the sum of ~N independent 2^-17-relative operand roundings, i.e. by ~sqrt(N) * 3e-5 * scale in absolute terms,
    # which is 1e-4 of a near-zero sum but 1e-7 of the mean; the round-1 form of this check compared raw sums at 1e-5.)
    count = ref.numel() / 32
    d_mean = ((st_ps[..., 0] - st_ref[..., 0]).abs() / count).max().item()
    d_msq = ((st_ps[..., 1] - st_ref[..., 1]).abs() / st_ref[..., 1].abs()).max().item()
    want_st = torch.stack([ref.view(1, -1, 32, Cout // 32).double().sum((1, 3)), (ref.view(1, -1, 32, Cout // 32).double() ** 2).sum((1, 3))], -1)
    d_own = ((st_ref - want_st).abs() / want_st.abs().clamp_min(1.0)).max().item()
    print(f"[upconv statistics] group mean differs by {d_mean:.2e}, mean square by {d_msq:.2e} (relative); plain kernel's statistics vs "
          f"fp64 sums of its own output {d_own:.2e}")
    assert d_mean < 1e-6 * max(1.0, scale) and d_msq < 1e-5
    if S <= 64:   # and against torch fp32 on the CPU
        xr = torch.relu(x[0, 0].permute(2, 0, 1)[None].cpu())
        want = F_conv_up(xr, w, b.cpu(), res)
        assert (out[0, 0].permute(2, 0, 1)[None].cpu() - want).abs().max().item() < 2e-4 * max(1.0, scale)


def F_conv_up(xr, w, b, res):
    import torch.nn.functional as F

    y = F.conv2d(F.interpolate(xr.double(), scale_factor=2, mode="nearest"), w.double(), b.double(), padding=1)
    if res is not None:
        y = y + F.interpolate(res[0, 0].permute(2, 0, 1)[None].cpu().double(), scale_factor=2, mode="nearest")
    return y.float()


def test_default_model_uses_the_folded_forms_and_agrees_with_the_plain_ones(ctx):
    """The shipped path runs the sub-pixel up-convolutions, the 4x4 stride-2 down-convolutions and fp16 two-plane networks
    (parity vs the reference: tests/test_model_gpu.py).  The plain forms they replace (nearest-x2 planes + 3x3 conv,
    conv + avgpool, three bf16 planes) stay reachable for shapes the folded kernels do not take; built explicitly here,
    they must give the same image up to the documented operand rounding."""
    from emoportraits_b200 import nets, ops
    from emoportraits_b200.infer import Model

    m = ctx["model"]
    assert m.decoder_nw.img[0].c1_ps is not None      # (the 160 -> 96 up block of the 256^2 config keeps the plain form: Cin % 64)
    assert all(b.c2_pool is not None for b in m.local_encoder_nw.blocks)
    assert m.precision["warp"] == ops.H2 and m.precision["decoder"] == 2
    plain = Model(ctx["cfg"], ctx["sd"], ctx["hsd"], "cuda", precision={k: 3 for k in m.precision if k != "decoder"})
    for b in plain.decoder_nw.img:
        b.c1_ps = None
    for b in plain.local_encoder_nw.blocks:
        b.c2_pool = None
    st = plain.source_pass(ctx["src"])
    img, _, _, so = plain.driver_pass(st, ctx["drv"][0], mix=True)
    _check(ctx["gold"]["default"], img, so, "plain forms (three bf16 planes, unfolded convolutions)")
    base, _, _, so0 = m.driver_pass(ctx["st"], ctx["drv"][0], mix=True)
    print(f"[default vs plain forms] image max-abs {(img - base).abs().max().item():.2e} "
          f"pose_embed {(so.target_pose_embed - so0.target_pose_embed).abs().max().item():.2e}")


# ------------------------------------------------------------------------------------------------------------------
# `3x3 conv -> 2x2 average pool` folded into one 4x4 stride-2 convolution (ops.fold_poolconv_weight; the form the
# down-sampling blocks run).  No kernel change: the implicit-GEMM kernel is generic in the tap count.
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Cin,Cout,S,planes", [(128, 128, 64, 2), (256, 256, 128, 2), (128, 256, 32, 3)])
def test_poolconv_fold_matches_conv_then_avgpool(Cin, Cout, S, planes):
    import math

    import torch.nn.functional as F

    from emoportraits_b200 import ops

    g = torch.Generator().manual_seed(Cin + S + planes)
    x = torch.randn((1, Cin, S, S), generator=g)
    w = torch.randn((Cout, Cin, 3, 3), generator=g) / math.sqrt(9 * Cin)
    b = torch.randn(Cout, generator=g)
    skip = torch.randn((1, Cout, S // 2, S // 2), generator=g)
    want = (F.avg_pool2d(F.conv2d(x.double(), w.double(), b.double(), padding=1), 2) + skip.double()).float()
    ops.begin_pass("cuda")
    a = ops.split_bf16(x.permute(0, 2, 3, 1)[:, None].contiguous().cuda(), planes)
    st = ops.new_stats(1, 32, "cuda")
    out = ops.conv_igemm(a, ops.pack_conv_weight(ops.fold_poolconv_weight(w), planes=planes), stride=(1, 2, 2), pad=(0, 1, 1),
                         bias=b.cuda(), residual=skip.permute(0, 2, 3, 1)[:, None].contiguous().cuda(), stats=st)
    torch.cuda.synchronize()
    got = out[:, 0].permute(0, 3, 1, 2).cpu()
    err = (got - want).abs().max().item()
    print(f"\n[4x4 stride-2 fold vs conv3x3 -> avgpool] {Cin}->{Cout} @{S}^2 planes {planes}: max-abs {err:.2e}")
    assert err < (2e-4 if planes == 2 else 2e-5) * max(1.0, want.abs().max().item())
    # statistics of the result, as the next GroupNorm needs them
    grp = want.view(1, 32, -1)
    ref_st = torch.stack([grp.double().sum(-1), (grp.double() ** 2).sum(-1)], -1)
    assert ((st.cpu() - ref_st).abs() / ref_st.abs().clamp_min(1.0)).max().item() < 1e-3


# ------------------------------------------------------------------------------------------------------------------
# fp16 two-plane operand mode ("h2", ops.H2; the default of every network but the decoder, infer.Model.PRECISION): three MMAs per
# product at fp32-level operand accuracy (tools/split_precision_emulation.py), meant to replace the six-MMA three-plane
# bf16 mode of the embedding / warp / source networks.
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Cin,Cout,sp,k", [(512, 512, (64, 64), 3), (96, 96, (16, 16), 3), (64, 32, (8, 16, 16), 3), (64, 128, (8, 8), 3),
                                           (256, 128, (8, 8, 8), 1)])
def test_conv_igemm_fp16_two_planes(Cin, Cout, sp, k):
    """same cases and bar as tests/test_ops_gpu.py::test_conv_igemm_three_planes: fp32-faithful against an fp64 reference"""
    import math

    import torch.nn.functional as F

    from emoportraits_b200 import ops

    g = torch.Generator().manual_seed(Cin + Cout)
    three_d = len(sp) == 3
    x = torch.randn(1, Cin, *sp, generator=g)
    w = torch.randn(Cout, Cin, *([k] * len(sp)), generator=g) / math.sqrt(Cin * k ** len(sp))
    b = torch.randn(Cout, generator=g)
    ref = (F.conv3d if three_d else F.conv2d)(x.double(), w.double(), b.double(), padding=k // 2)
    xc = x.permute(0, 2, 3, 4, 1).contiguous() if three_d else x.permute(0, 2, 3, 1)[:, None].contiguous()
    ops.begin_pass("cuda")
    a = ops.split_bf16(xc.cuda(), ops.H2)
    assert a.f16 and a.hi.dtype == torch.float16
    assert (a.float().cpu() - xc).abs().max().item() < 1e-5                # the planes reproduce the activations
    out = ops.conv_igemm(a, ops.pack_conv_weight(w, planes=ops.H2), bias=b.cuda())
    torch.cuda.synchronize()
    got = out.permute(0, 4, 1, 2, 3).cpu() if three_d else out[:, 0].permute(0, 3, 1, 2).cpu()
    err = (got.double() - ref).abs().max().item()
    print(f"\n[conv fp16 two planes vs fp64] {Cin}->{Cout} {sp} k{k}: max-abs {err:.2e} (scale {ref.abs().max().item():.2f})")
    assert err < 2e-5 * max(1.0, ref.abs().max().item())
    # GroupNorm + ReLU planes written by the apply pass in the same format
    st = ops.gn_stats(out, 32)
    gamma, beta = torch.rand(Cout, generator=g) + 0.5, torch.randn(Cout, generator=g)
    sp_h = ops.apply(out, gn=dict(stats=st, count=out.numel() / 32, gamma=gamma.cuda(), beta=beta.cuda()), act=ops.ACT_RELU, planes=ops.H2)
    want = torch.relu(F.group_norm(got, 32, gamma, beta, 1e-5))
    back = sp_h.float().permute(0, 4, 1, 2, 3).cpu() if three_d else sp_h.float()[:, 0].permute(0, 3, 1, 2).cpu()
    assert (back - want).abs().max().item() < 1e-4
