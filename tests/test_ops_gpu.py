"""GPU unit tests of every C-ABI op against a plain PyTorch fp32 CPU reference of the same op."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def cl(x):  # NCDHW/NCHW -> channels-last (N,D,H,W,C)
    if x.dim() == 4:
        x = x[:, :, None]
    return x.permute(0, 2, 3, 4, 1).contiguous()


def uncl(x):  # (N,D,H,W,C) -> NCDHW
    return x.permute(0, 4, 1, 2, 3).contiguous()


@pytest.fixture(scope="module")
def ops():
    from emoportraits_b200 import ops as o
    return o


def _grid(N, D, H, W, seed, jitter=0.1, rot=False):
    g = torch.Generator().manual_seed(seed)
    zs, ys, xs = torch.linspace(-1, 1, D), torch.linspace(-1, 1, H), torch.linspace(-1, 1, W)
    w, v, u = torch.meshgrid(zs, ys, xs, indexing="ij")
    base = torch.stack([u, v, w], -1)[None].repeat(N, 1, 1, 1, 1)
    grid = base + jitter * torch.randn(base.shape, generator=g)
    if rot:
        a = math.radians(30)
        R = torch.tensor([[math.cos(a), -math.sin(a), 0], [math.sin(a), math.cos(a), 0], [0, 0, 1.0]])
        grid = grid @ R.T + 0.2
    return grid.contiguous()


@pytest.mark.parametrize("shape", [(1, 96, 16, 64, 64), (2, 8, 5, 7, 9), (1, 96, 64, 64, 64)])
@pytest.mark.parametrize("rot", [False, True])
def test_grid_sample3d_ncdhw(ops, shape, rot):
    N, C, D, H, W = shape
    x = torch.randn(shape, generator=torch.Generator().manual_seed(0))
    grid = _grid(N, D, H, W, 1, rot=rot)
    ref = F.grid_sample(x, grid, mode="bilinear", padding_mode="zeros", align_corners=False)
    out = ops.grid_sample3d(x.cuda(), grid=grid.cuda(), in_layout="ncdhw").cpu()
    assert out.shape == ref.shape
    assert (out - ref).abs().max().item() < 2e-5


@pytest.mark.parametrize("shape", [(1, 96, 16, 64, 64), (2, 8, 5, 7, 9)])
@pytest.mark.parametrize("out_layout", ["cl", "hwdc", "ncdhw"])
def test_grid_sample3d_channels_last(ops, shape, out_layout):
    N, C, D, H, W = shape
    x = torch.randn(shape, generator=torch.Generator().manual_seed(0))
    grid = _grid(N, D, H, W, 2, rot=True)
    ref = F.grid_sample(x, grid, mode="bilinear", padding_mode="zeros", align_corners=False)
    out, sp = ops.grid_sample3d(cl(x).cuda(), grid=grid.cuda(), in_layout="cl", out_layout=out_layout, want_split=True)
    out, rec = out.cpu(), sp.float().cpu()
    if out_layout == "cl":
        out, rec = uncl(out), uncl(rec)
    elif out_layout == "hwdc":
        out, rec = out.permute(0, 4, 3, 1, 2), rec.permute(0, 4, 3, 1, 2)
    assert (out - ref).abs().max().item() < 2e-5
    assert (rec - ref).abs().max().item() < 2e-5 + ref.abs().max().item() * 2 ** -16


def test_grid_sample3d_affine_matches_bmm_grid(ops):
    """theta variant == identity_grid_3d.bmm(theta[:, :3]^T) then F.grid_sample (infer.py:441-444, 583-588)."""
    N, C, D, S = 2, 96, 16, 64
    x = torch.randn(N, C, D, S, S, generator=torch.Generator().manual_seed(3))
    a, b = math.radians(12), math.radians(-7)
    th = torch.tensor([[[math.cos(a), -math.sin(a), 0.05, 0.03], [math.sin(a), math.cos(a), -0.02, -0.04], [0.01, 0.03, 1.1, 0.02]],
                       [[0.9 * math.cos(b), -math.sin(b), 0.0, 0.4], [math.sin(b), 0.9 * math.cos(b), 0.1, -0.3], [0.0, -0.1, 0.8, 0.1]]])
    gs, gz = torch.linspace(-1, 1, S), torch.linspace(-1, 1, D)
    w, v, u = torch.meshgrid(gz, gs, gs, indexing="ij")
    idg = torch.stack([u, v, w, torch.ones_like(u)], 3).view(1, -1, 4).repeat(N, 1, 1)
    grid = idg.bmm(th.transpose(1, 2)).view(N, D, S, S, 3)
    ref = F.grid_sample(x, grid, padding_mode="zeros", align_corners=False)
    out = ops.grid_sample3d(x.cuda(), theta=th.cuda(), out_size=(D, S, S), in_layout="ncdhw").cpu()
    assert (out - ref).abs().max().item() < 1e-4
    out2 = uncl(ops.grid_sample3d(cl(x).cuda(), theta=th.cuda(), out_size=(D, S, S), in_layout="cl").cpu())
    assert (out2 - ref).abs().max().item() < 1e-4


def test_grid_sample2d_affine_and_resize(ops):
    img = torch.rand(2, 3, 64, 64, generator=torch.Generator().manual_seed(0))
    th = torch.tensor([[[0.5, 0.05, 0.1], [-0.04, 0.55, -0.05]], [[0.45, 0.0, 0.0], [0.0, 0.45, 0.2]]])
    g = torch.linspace(-1, 1, 32)
    v, u = torch.meshgrid(g, g, indexing="ij")
    idg = torch.stack([u, v, torch.ones_like(u)], 2).view(1, -1, 3).repeat(2, 1, 1)
    grid = idg.bmm(th.transpose(1, 2)).view(2, 32, 32, 2)
    ref = F.grid_sample(img, grid, align_corners=False)
    mean, std = torch.tensor([0.485, 0.456, 0.406]), torch.tensor([0.229, 0.224, 0.225])
    out, nchw = ops.grid_sample2d_affine(img.cuda(), th.cuda(), (32, 32), mean.cuda(), std.cuda(), want_nchw=True)
    assert (nchw.cpu() - ref).abs().max().item() < 1e-5
    refn = (ref - mean[None, :, None, None]) / std[None, :, None, None]
    got = out.cpu()[:, 0].permute(0, 3, 1, 2)
    assert (got[:, :3] - refn).abs().max().item() < 1e-5 and got[:, 3].abs().max().item() == 0
    ref2 = F.interpolate(img, size=(16, 16), mode="bilinear")
    got2 = ops.resize_bilinear(img.cuda(), (16, 16)).cpu()[:, 0].permute(0, 3, 1, 2)[:, :3]
    assert (got2 - ref2).abs().max().item() < 1e-6


@pytest.mark.parametrize("C,shape", [(512, (1, 64, 64)), (96, (16, 16, 16)), (320, (1, 32, 32)), (32, (4, 8, 8))])
def test_groupnorm_relu_apply(ops, C, shape):
    N = 2
    g = torch.Generator().manual_seed(0)
    x = torch.randn(N, C, *shape, generator=g) * 2 + 0.5
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    ref = F.relu(F.group_norm(x, 32, gamma, beta, 1e-5))
    xc = cl(x).cuda()
    st = ops.gn_stats(xc, 32)
    A, B = ops.gn_finalize(st, x[0].numel() / 32, gamma.cuda(), beta.cuda())
    out, sp = ops.apply(xc, A, B, act=ops.ACT_RELU, want_f32=True, want_split=True)
    assert (uncl(out.cpu()) - ref).abs().max().item() < 2e-5
    assert (uncl(sp.float().cpu()) - ref).abs().max().item() < 2e-5 + ref.abs().max().item() * 2 ** -16


def test_apply_upsample_and_residual(ops):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1, 64, 8, 8, generator=g)
    r = torch.randn(1, 64, 8, 8, generator=g)
    A, B = torch.randn(1, 64, generator=g), torch.randn(1, 64, generator=g)
    ref = F.interpolate(F.relu(x * A[0][None, :, None, None] + B[0][None, :, None, None] + r), scale_factor=2, mode="nearest")
    out = ops.apply(cl(x).cuda(), A.cuda(), B.cuda(), act=ops.ACT_RELU, res=cl(r).cuda(), up=2, want_f32=True, want_split=False)
    assert (uncl(out.cpu())[:, :, 0] - ref).abs().max().item() < 1e-6


def _conv_case(ops, N, Cin, Cout, sp, k, stride=1, bias=True, residual=False, act=0, stats=False, out_nchw=False, seed=0,
               planes=2, split_k=True, res_shift=0):
    g = torch.Generator().manual_seed(seed)
    three_d = len(sp) == 3
    x = torch.randn(N, Cin, *sp, generator=g)
    w = torch.randn(Cout, Cin, *([k] * len(sp)), generator=g) / math.sqrt(Cin * k ** len(sp))
    b = torch.randn(Cout, generator=g) if bias else None
    conv = F.conv3d if three_d else F.conv2d
    ref = conv(x.double(), w.double(), b.double() if bias else None, stride=stride, padding=k // 2)
    res = None
    if residual:
        if res_shift:   # residual at half the output resolution, read with nearest-neighbour replication (2-D maps)
            res = torch.randn(ref.shape[:2] + tuple(v // 2 for v in ref.shape[2:]), generator=g)
            ref = ref + F.interpolate(res.double(), scale_factor=2, mode="nearest")
        else:
            res = torch.randn(ref.shape, generator=g)
            ref = ref + res.double()
    if act == 2:
        ref = torch.sigmoid(ref)
    elif act == 3:
        ref = torch.tanh(ref)
    pw = ops.pack_conv_weight(w, planes=planes)
    a = ops.split_bf16(cl(x).cuda(), planes)
    st = ops.new_stats(N, 32, "cuda") if stats else None
    s3 = (stride,) * 3 if three_d else (1, stride, stride)
    out = ops.conv_igemm(a, pw, stride=s3, bias=b.cuda() if bias else None, residual=cl(res).cuda() if residual else None,
                         act=act, stats=st, out_nchw=out_nchw, split_k=split_k, res_shift=res_shift)
    torch.cuda.synchronize()
    got = out.cpu() if out_nchw else uncl(out.cpu())
    if not three_d:
        got = got[:, :, 0]
    scale = ref.abs().max().item()
    err = (got.double() - ref).abs().max().item()
    print(f"[conv {N}x{Cin}->{Cout} {sp} k{k} s{stride}] max-abs err {err:.2e} (ref max {scale:.2e}, rel {err / scale:.1e})")
    assert err < 2e-5 * max(scale, 1.0), (err, scale)
    if stats:
        r = ref.float().reshape(N, 32, -1)
        s_ref = torch.stack([r.double().sum(-1), (r.double() ** 2).sum(-1)], -1)
        assert torch.allclose(st.cpu(), s_ref, rtol=1e-4, atol=1e-2), (st.cpu() - s_ref).abs().max()
    return err


@pytest.mark.parametrize("Cin,Cout,sp,k", [
    (64, 64, (16, 16), 3),        # one k-chunk of 64, single tile
    (128, 128, (32, 32), 3),      # multiple tiles
    (512, 512, (64, 64), 3),      # decoder res block shape
    (512, 320, (32, 32), 3),      # N tile 160
    (192, 128, (32, 32), 3),
    (96, 96, (16, 16), 3),        # KC = 32 path (SWIZZLE_64B)
    (1536, 512, (64, 64), 1),     # decoder input 1x1
    (128, 3, (32, 32), 1),        # ragged Cout head
    (32, 32, (8, 8), 3),
])
def test_conv2d_igemm(ops, Cin, Cout, sp, k):
    _conv_case(ops, 1, Cin, Cout, sp, k, bias=True, residual=(Cout % 4 == 0), stats=(Cout % 32 == 0))


@pytest.mark.parametrize("Cin,Cout,sp,k", [(512, 512, (64, 64), 3), (96, 96, (16, 16), 3), (512, 256, (8, 8, 8), 3), (64, 128, (8, 8), 3)])
def test_conv_igemm_three_planes(ops, Cin, Cout, sp, k):
    """fp32-faithful mode (hi, lo, lo2 planes, six MMAs per product)"""
    err = _conv_case(ops, 1, Cin, Cout, sp, k, bias=True, residual=True, stats=True, planes=3)


@pytest.mark.parametrize("N,Cin,Cout,sp,k,planes,kw", [
    (1, 64, 96, (24, 40), 3, 2, dict(residual=True, stats=True)),          # ragged pixel boxes: conv<64,2> BN16 rr3, per-column statistics
    (1, 64, 128, (256, 256), 3, 2, dict(residual=False, stats=True)),      # no residual, several tiles per CTA: conv<64,2> BN128 rr2
    (1, 512, 320, (32, 32), 3, 2, dict(residual=True, stats=True)),        # 20 N tiles of 16 (BN narrowed from 80 on 8 pixel tiles)
    (2, 64, 96, (16, 32), 3, 2, dict(residual=True, stats=True, act=3)),   # batch of 2 (per-sample statistics), tanh
    (1, 64, 128, (32, 32), 3, 2, dict(residual=True, res_shift=1, stats=True)),  # half-resolution residual: quarter-size TMA tile
    (1, 64, 128, (24, 40), 3, 2, dict(residual=True, res_shift=1, stats=True)),  # the same on ragged tiles
    (1, 64, 96, (4, 16, 16), 3, 3, dict(residual=True, stats=True)),       # 3-D volume (tiles inside one depth slice), three planes
    (1, 96, 96, (4, 16, 16), 3, "h2", dict(residual=True, stats=True)),    # fp16 planes, KC = 32
    (1, 256, 128, (32, 32), 1, 2, dict(residual=True, stats=False)),       # 1x1 (per-tap main loop)
])
def test_conv_igemm_tma_epilogue(ops, N, Cin, Cout, sp, k, planes, kw):
    """The residual / statistics final phase and the row-reuse main loop on small shapes the model would hand to split-K:
    forced here with split_k=False.  (The name is kept so that the test ids stay stable: the TMA-store epilogue it was written
    for no longer exists, and these shapes now exercise the register final phase.)"""
    _conv_case(ops, N, Cin, Cout, sp, k, bias=True, planes=planes, split_k=False, **kw)


@pytest.mark.parametrize("N,Cin,Cout,sp,mode,planes", [
    (1, 64, 64, (32, 32), "gn", "h2"),        # ResNet-18 layer1 shape: split-K, fused finalize + GroupNorm + ReLU + fp16 planes
    (1, 256, 512, (4, 4), "gn_res", "h2"),    # layer4: 16 pixels, 18 K parts; residual + fp32 + planes out
    (2, 128, 128, (16, 16), "bn_res", 2),     # eval-BatchNorm affine, batch of 2, bf16 planes
    (1, 64, 64, (8, 8, 8), "gn", 3),          # small 3-D layer, three planes
    (1, 128, 128, (64, 64), "gn", 2),         # too large for the fused finalize: convolution + elementwise pass (same result)
])
def test_conv_post_op(ops, N, Cin, Cout, sp, mode, planes):
    """conv_igemm(..., post=...) == conv -> norm -> (+ residual) -> ReLU of torch in fp64, whichever way the library runs it
    (emo_conv_desc.post), and the fused split-K path is bit-reproducible run to run (fixed summation orders)."""
    g = torch.Generator().manual_seed(Cin + Cout)
    three_d = len(sp) == 3
    x = torch.randn(N, Cin, *sp, generator=g)
    w = torch.randn(Cout, Cin, *([3] * len(sp)), generator=g) / math.sqrt(Cin * 3 ** len(sp))
    b = torch.randn(Cout, generator=g)
    conv = F.conv3d if three_d else F.conv2d
    y = conv(x.double(), w.double(), b.double(), padding=1)
    gamma, beta = torch.rand(Cout, generator=g) + 0.5, torch.randn(Cout, generator=g)
    res = torch.randn(y.shape, generator=g) if mode.endswith("res") else None
    bshape = (1, Cout) + (1,) * len(sp)
    if mode.startswith("gn"):
        z = F.group_norm(y, 32, gamma.double(), beta.double(), 1e-5)
    else:
        z = y * gamma.double().view(bshape) + beta.double().view(bshape)
    if res is not None:
        z = z + res.double()
    ref = torch.relu(z).float()
    a = ops.split_bf16(cl(x).cuda(), planes)
    pw = ops.pack_conv_weight(w, planes=planes)

    def run():
        ops.begin_pass("cuda")
        st = ops.new_stats(N, 32, "cuda") if mode.startswith("gn") else None
        post = dict(act=ops.ACT_RELU, planes=planes, want_f32=True, want_split=True, res=cl(res).cuda() if res is not None else None)
        if mode.startswith("gn"):
            post["gn"] = dict(stats=st, count=y.numel() / N / 32, gamma=gamma.cuda(), beta=beta.cuda())
        else:
            post.update(A=gamma[None].cuda().contiguous(), B=beta[None].cuda().contiguous(), per_sample=False)
        out, sp_ = ops.conv_igemm(a, pw, bias=b.cuda(), stats=st, post=post)
        torch.cuda.synchronize()
        return out, sp_

    out, planes_out = run()
    got = uncl(out.cpu())
    got = got if three_d else got[:, :, 0]
    err = (got - ref).abs().max().item()
    perr = ((uncl(planes_out.float().cpu()) if three_d else uncl(planes_out.float().cpu())[:, :, 0]) - ref).abs().max().item()
    print(f"\n[conv post-op {mode} {N}x{Cin}->{Cout} {sp} planes {planes}] fp32 out err {err:.2e}, planes err {perr:.2e} (ref max {ref.abs().max().item():.2f})")
    assert err < 5e-5 * max(1.0, ref.abs().max().item())
    assert perr < (2e-4 if planes == 2 else 5e-5) * max(1.0, ref.abs().max().item())
    out2, planes2 = run()
    if y.numel() // N <= 65536:      # the fused split-K path: fixed summation orders
        assert torch.equal(out, out2) and torch.equal(planes_out.hi, planes2.hi) and torch.equal(planes_out.lo, planes2.lo)


def test_conv_statistics_are_reproducible(ops):
    """GroupNorm statistics of a multi-tile layer: per-tile column sums go through per-quadrant slots (one writer each, fixed
    summation order), the per-tile group sums are added to the global fp64 sums with atomics - fp64 sums of fp32-sized terms,
    whose order can only move the last bits of a double: two runs agree to 1e-13 relative (the shared-memory fp32 atomics of
    round 1 left 1e-7; see test_resampler_statistics_are_reproducible for the other producers of statistics)."""
    g = torch.Generator().manual_seed(11)
    x = torch.randn(1, 1, 128, 128, 128, generator=g).cuda()
    w = torch.randn(128, 128, 3, 3, generator=g) / math.sqrt(9 * 128)
    a, pw = ops.split_bf16(x, 2), ops.pack_conv_weight(w)
    res = torch.randn(1, 1, 128, 128, 128, generator=g).cuda()
    outs = []
    for _ in range(3):
        ops.begin_pass("cuda")
        st = ops.new_stats(1, 32, "cuda")
        y = ops.conv_igemm(a, pw, residual=res, stats=st)
        torch.cuda.synchronize()
        outs.append((y.clone(), st.clone()))
    for y, st in outs[1:]:
        assert torch.equal(y, outs[0][0])
        rel = ((st - outs[0][1]).abs() / outs[0][1].abs().clamp_min(1e-30)).max().item()
        assert rel < 1e-13, rel


def test_conv2d_igemm_batch_and_act(ops):
    _conv_case(ops, 2, 128, 3, (32, 32), 1, act=2, out_nchw=True)
    _conv_case(ops, 2, 64, 64, (16, 16), 3, act=3)


@pytest.mark.parametrize("Cin,Cout,sp,k", [
    (64, 32, (4, 16, 16), 3),
    (96, 96, (4, 16, 16), 3),
    (512, 256, (8, 8, 8), 3),
    (32, 3, (4, 16, 16), 3),
    (64, 128, (4, 8, 8), 1),
])
def test_conv3d_igemm(ops, Cin, Cout, sp, k):
    _conv_case(ops, 1, Cin, Cout, sp, k, bias=True, residual=(Cout % 4 == 0), stats=(Cout % 32 == 0))


@pytest.mark.parametrize("sp", [(32, 32), (8, 8)])
def test_conv2d_igemm_stride2(ops, sp):
    _conv_case(ops, 1, 64, 128, sp, 3, stride=2, bias=False)
    _conv_case(ops, 1, 64, 128, sp, 1, stride=2, bias=False)


def test_wrapper_boundary_image_ops(ops):
    """uint8 <-> fp32 image conversion and the bicubic pre-processing resize against the torch ops the reference calls
    (ToTensor / clamp + ToPILImage: notebooks/infer.py:229-243, 641-644; F.interpolate bicubic :399-403)"""
    g = torch.Generator().manual_seed(3)
    u8 = torch.randint(0, 256, (2, 37, 53, 3), generator=g, dtype=torch.uint8)
    got = ops.u8_to_image(u8.cuda()).cpu()
    assert torch.equal(got, u8.permute(0, 3, 1, 2).float().div(255))
    x = torch.rand(2, 3, 40, 24, generator=g) * 1.4 - 0.2                      # values outside [0, 1] are clamped
    x[0, 0, 0, :4] = torch.tensor([1.0, 0.0, 0.999999, 254.5 / 255.0])
    want = (x.clamp(0, 1) * 255).byte().permute(0, 2, 3, 1)
    assert torch.equal(ops.image_to_u8(x.cuda()).cpu(), want)
    img, mask, bg = torch.rand(2, 3, 20, 28, generator=g), torch.rand(2, 1, 20, 28, generator=g), torch.rand(3, 20, 28, generator=g)
    m8 = torch.where(mask > 0.3, mask, mask * 0) ** 8          # E_emo_infer_video.ipynb cell 41
    got = ops.composite(img.cuda(), mask.cuda(), bg.cuda()).cpu()
    assert (got - (m8 * img + (1 - m8) * bg[None])).abs().max().item() < 1e-6
    for (hi, wi, ho, wo) in [(300, 280, 256, 256), (128, 160, 256, 512), (512, 512, 256, 256)]:
        y = torch.rand(1, 3, hi, wi, generator=g)
        ref = F.interpolate(y, size=(ho, wo), mode="bicubic")
        err = (ops.resize_bicubic(y.cuda(), (ho, wo)).cpu() - ref).abs().max().item()
        print(f"[bicubic {hi}x{wi} -> {ho}x{wo}] max-abs err vs F.interpolate {err:.2e}")
        assert err < 2e-6


def test_conv_direct_stem(ops):
    g = torch.Generator().manual_seed(0)
    x = torch.rand(1, 3, 64, 64, generator=g)
    w = torch.randn(128, 3, 7, 7, generator=g) * 0.1
    b = torch.randn(128, generator=g)
    ref = F.conv2d(x, w, b, padding=3)
    xc = torch.zeros(1, 1, 64, 64, 4)
    xc[..., :3] = cl(x)
    wc = torch.zeros(7, 7, 4, 128)
    wc[:, :, :3] = w.permute(2, 3, 1, 0)
    st = ops.new_stats(1, 32, "cuda")
    out = ops.conv_direct(xc.cuda(), wc.cuda(), 1, 3, b.cuda(), stats=st)
    assert (uncl(out.cpu())[:, :, 0] - ref).abs().max().item() < 1e-4
    r = ref.reshape(1, 32, -1).double()
    assert torch.allclose(st.cpu(), torch.stack([r.sum(-1), (r ** 2).sum(-1)], -1), rtol=1e-4, atol=1e-2)
    ref2 = F.conv2d(x, w[:64], None, stride=2, padding=3)
    out2 = ops.conv_direct(xc.cuda(), wc[..., :64].contiguous().cuda(), 2, 3)
    assert (uncl(out2.cpu())[:, :, 0] - ref2).abs().max().item() < 1e-4


def test_linear(ops):
    g = torch.Generator().manual_seed(0)
    x, w, b = torch.randn(3, 128, generator=g), torch.randn(70, 128, generator=g), torch.randn(70, generator=g)
    add = torch.randn(3, 70, generator=g)
    ref = (x @ w.T + b + add) * 0.5
    out = ops.linear(x.cuda(), w.cuda(), b.cuda(), add.cuda(), scale=0.5).cpu()
    assert (out - ref).abs().max().item() < 1e-4


@pytest.mark.parametrize("f", [(2, 2, 2), (1, 2, 2), (2, 1, 1)])
def test_resamples(ops, f):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 64, 4, 6, 8, generator=g)
    ref = F.interpolate(x, scale_factor=f, mode="trilinear")
    st = ops.new_stats(2, 32, "cuda")
    out = ops.upsample_trilinear(cl(x).cuda(), f, stats=st)
    assert (uncl(out.cpu()) - ref).abs().max().item() < 1e-5
    r = ref.reshape(2, 32, -1).double()
    assert torch.allclose(st.cpu(), torch.stack([r.sum(-1), (r ** 2).sum(-1)], -1), rtol=1e-4, atol=1e-2)
    ref2 = F.avg_pool3d(x, kernel_size=f, stride=f)
    out2 = ops.avgpool(cl(x).cuda(), f)
    assert (uncl(out2.cpu()) - ref2).abs().max().item() < 1e-5


def test_maxpool_and_global_avgpool(ops):
    x = torch.randn(2, 64, 16, 16, generator=torch.Generator().manual_seed(0))
    ref = F.max_pool2d(x, 3, 2, 1)
    out = ops.maxpool2d_3x3s2(cl(x).cuda())
    assert (uncl(out.cpu())[:, :, 0] - ref).abs().max().item() == 0
    assert (ops.global_avgpool(cl(x).cuda()).cpu() - x.mean((2, 3))).abs().max().item() < 1e-5


def test_pose_theta(ops):
    """smoke test of ops.pose_theta against the oracle; tests/test_pose_kernel_gpu.py checks the kernel in every mode"""
    from oracle import restatement as R
    srt = torch.tensor([[1.0, 1.1, 0.9, 0.15, -0.1, 0.05, 0.03, -0.02, 0.01], [0.8, 0.9, 1.0, -0.3, 0.2, 0.1, -0.1, 0.05, 0.0]])
    th_ref = R.get_transform_matrix(srt[:, :3], srt[:, 3:6], srt[:, 6:])
    th, warp, align = ops.pose_theta(srt.cuda(), invert_warp=True)
    assert (th.cpu() - th_ref).abs().max().item() < 1e-6
    assert (warp.cpu() - th_ref.inverse()[:, :3]).abs().max().item() < 1e-5
    src = th_ref[0]
    mixed_ref = R.get_mixing_theta(src[None], th_ref[1:2])
    th2, warp2, align2 = ops.pose_theta(srt[1:2].cuda(), source_theta=src.cuda().contiguous(), mix=True)
    assert (th2.cpu()[:, :3] - mixed_ref).abs().max().item() < 1e-5
    assert (align2.cpu() - R.align_theta_2d(mixed_ref)).abs().max().item() < 1e-5


def test_stats_arena_is_keyed_by_resolved_device(ops):
    """begin_pass() gets the model's device ('cuda'), new_stats() a tensor's ('cuda:0'): both must name the same arena,
    otherwise a captured frame accumulates into slices that its own begin_pass never zeroes (regression: the second
    replay of a graph captured after another model had used the 'cuda:0' spelling returned garbage)."""
    import torch
    ops.begin_pass(torch.device("cuda"))
    t = ops.new_stats(1, 32, torch.zeros(1, device="cuda").device)
    buf = ops._ARENA[(ops._dev_key("cuda"), ops._SLOT)]["buf"]
    assert buf.data_ptr() <= t.data_ptr() < buf.data_ptr() + buf.numel() * 8
    prev = ops.set_slot(1)
    try:
        ops.begin_pass("cuda:0")
        t1 = ops.new_stats(1, 32, "cuda")
        assert t1.data_ptr() != t.data_ptr()
    finally:
        ops.set_slot(prev)


@pytest.mark.parametrize("C,Cout,S,act", [(128, 3, (64, 64), "sigmoid"), (128, 3, (37, 21), "none"), (256, 4, (16, 16), "sigmoid"), (32, 1, (8, 8), "none")])
def test_gn_head(ops, C, Cout, S, act):
    """image head: act(bias + w . relu(GroupNorm(x))) in one pass == torch group_norm -> relu -> 1x1 conv -> act"""
    import torch
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(5)
    N = 2
    x = (torch.randn(N, 1, *S, C, generator=g) * 1.7 + 0.3).cuda()
    gamma, beta = (torch.rand(C, generator=g) + 0.5).cuda(), torch.randn(C, generator=g).cuda()
    w, b = (torch.randn(Cout, C, generator=g) / C ** 0.5).cuda(), torch.randn(Cout, generator=g).cuda()
    st = ops.gn_stats(x, 32)
    cnt = x.numel() / N / 32
    out = ops.gn_head(x, dict(stats=st, count=cnt, gamma=gamma, beta=beta), w, b,
                      act_out=ops.ACT_SIGMOID if act == "sigmoid" else ops.ACT_NONE)
    xr = x[:, 0].permute(0, 3, 1, 2).double()
    ref = F.conv2d(F.relu(F.group_norm(xr, 32, gamma.double(), beta.double(), 1e-5)), w.double()[:, :, None, None], b.double())
    if act == "sigmoid":
        ref = torch.sigmoid(ref)
    assert out.shape == (N, Cout, 1, *S)
    err = (out[:, :, 0].double() - ref).abs().max().item()
    assert err < 2e-5, err


# ------------------------------------------------------------------------------------------------------------------
# grid_sample_3d at BASELINE's largest size and its edge cases (validated kernels, new tests)
# ------------------------------------------------------------------------------------------------------------------
def test_grid_sample3d_full_size_batch32_properties():
    """BASELINE configs[2] at its largest size (96ch x 64^3 volume, 64^3 lattice, batch 32: 25.8 GB in, 25.8 GB out), where a
    CPU reference would take minutes: size-independent properties instead, all bit-exact.
      * batch independence: sample n of the batched call == the single-sample call on (x[n], theta[n] / grid[n]);
      * linearity in the volume for a power-of-two factor: gs(0.5 x) == 0.5 gs(x);
      * zeros padding: a lattice entirely outside the volume samples exactly 0;
      * channel equivariance: permuting the channels of the volume permutes the channels of the result."""
    from emoportraits_b200 import ops

    N, C, S = 32, 96, 64
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn((N, S, S, S, C), generator=g, device="cuda")
    ang = torch.linspace(-0.6, 0.6, N)
    th = torch.zeros(N, 3, 4)
    th[:, 0, 0], th[:, 0, 1], th[:, 1, 0], th[:, 1, 1], th[:, 2, 2] = ang.cos(), -ang.sin(), ang.sin(), ang.cos(), 0.9
    th[:, :, 3] = torch.tensor([0.2, -0.1, 0.05])
    th = th.cuda().contiguous()
    out = ops.grid_sample3d(x, theta=th, out_size=(S, S, S), in_layout="cl")
    assert out.shape == (N, S, S, S, C)
    for n in (0, 17, 31):
        one = ops.grid_sample3d(x[n:n + 1].contiguous(), theta=th[n:n + 1].contiguous(), out_size=(S, S, S), in_layout="cl")
        assert torch.equal(one[0], out[n]), n
    assert (out[31] != 0).float().mean().item() > 0.5            # a rotated, shifted lattice still lands mostly inside
    half = ops.grid_sample3d((x[:2] * 0.5).contiguous(), theta=th[:2].contiguous(), out_size=(S, S, S), in_layout="cl")
    assert torch.equal(half, out[:2] * 0.5)
    perm = torch.randperm(C, generator=torch.Generator().manual_seed(6)).cuda()
    pc = ops.grid_sample3d(x[:1, ..., perm].contiguous(), theta=th[:1].contiguous(), out_size=(S, S, S), in_layout="cl")
    assert torch.equal(pc, out[:1, ..., perm])
    far = th[:1].clone()
    far[:, :, 3] = 4.0
    assert ops.grid_sample3d(x[:1].contiguous(), theta=far.contiguous(), out_size=(S, S, S), in_layout="cl").abs().max().item() == 0.0
    del out, half, pc
    # explicit grid tensor (jittered identity lattice), batch 32
    grid = (_grid(1, S, S, S, 9).cuda() + 0.02 * torch.arange(N, device="cuda").view(N, 1, 1, 1, 1)).contiguous()
    outg = ops.grid_sample3d(x, grid=grid, in_layout="cl")
    for n in (0, 31):
        one = ops.grid_sample3d(x[n:n + 1].contiguous(), grid=grid[n:n + 1].contiguous(), in_layout="cl")
        assert torch.equal(one[0], outg[n]), n


def test_grid_sample3d_empty_and_invalid_inputs():
    """edge cases: an empty batch returns an empty tensor (as F.grid_sample does) without launching; malformed arguments
    are refused by the C-ABI with a message (EMO_ERR_INVALID -> RuntimeError), never launched."""
    from emoportraits_b200 import ops

    e = ops.grid_sample3d(torch.empty((0, 4, 4, 4, 8), device="cuda"), theta=torch.empty((0, 3, 4), device="cuda"),
                          out_size=(4, 4, 4), in_layout="cl")
    assert e.shape == (0, 4, 4, 4, 8)
    x = torch.randn((1, 4, 4, 4, 6), device="cuda")          # channels-last path needs C % 4 == 0
    with pytest.raises(RuntimeError, match="C % 4"):
        ops.grid_sample3d(x, theta=torch.eye(4, device="cuda")[None, :3].contiguous(), out_size=(4, 4, 4), in_layout="cl")




@pytest.mark.gpu
def test_resampler_statistics_are_reproducible(ops):
    """The GroupNorm statistics that are NOT produced by a convolution epilogue - trilinear up-sampling (+ add), average pooling,
    the stand-alone statistics pass, the un-fused split-K finalize - accumulate per CTA in fp64 shared memory (sums of fp32 terms
    are exact in fp64, whatever order the atomics arrive in) and then in the global fp64 sums: repeated runs agree to the last
    bits of a double, and both match an fp64 torch reduction of the produced tensor."""
    g = torch.Generator().manual_seed(13)
    x = torch.randn(1, 8, 16, 16, 128, generator=g).cuda() * 3 + 0.5
    add = torch.randn(1, 16, 32, 32, 128, generator=g).cuda()

    def ref(y):
        t = y.double().reshape(1, -1, 32, 4)  # [N][spatial][G][C/G]
        return torch.stack([t.sum((1, 3)), (t * t).sum((1, 3))], -1), torch.stack([t.abs().sum((1, 3)), (t * t).sum((1, 3))], -1)

    cases = {"upsample": lambda st: ops.upsample_trilinear(x, (2, 2, 2), add=add, stats=st),
             "avgpool": lambda st: ops.avgpool(add, (1, 2, 2), stats=st),
             "gn_stats": lambda st: (ops.gn_stats(add, 32, stats=st), add)[1]}
    for name, fn in cases.items():
        runs = []
        for _ in range(3):
            ops.begin_pass("cuda")
            st = ops.new_stats(1, 32, "cuda")
            y = fn(st)
            torch.cuda.synchronize()
            runs.append((y.clone(), st.clone()))
        want, scale = ref(runs[0][0])
        for y, st in runs:
            assert torch.equal(y, runs[0][0]), name
            assert ((st - runs[0][1]).abs() / runs[0][1].abs().clamp_min(1.0)).max().item() < 1e-13, name
            # per-thread partial sums are fp32 (a fixed order per thread), squares are rounded to fp32: ~1e-7 of the sum of magnitudes
            assert ((st.reshape(want.shape) - want).abs() / scale).max().item() < 2e-6, name
