"""GPU tests of the source pass's fast mode (InferenceWrapper(source_precision="fast"), Model.SOURCE_FAST): the local encoder,
the source volume blocks and the 3-D U-Net on one fp16 operand plane (ops.H1), and the local encoder's 7x7 RGB stem as a 7x1
implicit GEMM over ops.stem_pack's 32 channels that also writes the GroupNorm statistics of its output.

Op level, one case per one-plane plan class the fast source pass reaches in 3-D (3x3x3 at Cin = 96 on KC = 32, 192, 384 and
512; 1^3 skips and the U-Net head; residual; GroupNorm statistics; the GroupNorm post-op), a depth-tiled 3-D tile, and the
pool-folded 4x4 stride-2 encoder convolutions with statistics (tests/test_fast_source_cpu.py checks that these tables cover
every convolution of the fast source pass at 256^2 and 512^2).  Every output, the statistics included, is written into a
buffer followed by a NaN guard region:
  * within 1e-5 of the scale of float64 on the ROUNDED operands, fp16(x * 16) / 16 and fp16(w * 256) / 256;
  * within the one-plane operand bound 2^-10 conv(|x|, |w|) (+ 1e-5 of the scale) of float64 on the fp32 operands;
  * the statistics (per-group sum and sum of squares) against float64 of the rounded-operand result;
  * the GroupNorm + ReLU post-op in fp32 and its one fp16 plane within fp16 rounding of the float64 post-op.
The stem with statistics: against float64 on the rounded operands, against conv_direct (the exact mode's stem) within the
operand bound, and its statistics against float64.
Model level at 256^2 and 512^2 (synthetic seed-0 weights; tools/decoder_precision_emulation.py --source gives the bounds): the
unswitched source outputs are bit-identical to exact mode, target_latent_volume stays within its bound, two runs are
bit-identical, the largest activation any one-plane convolution reads has 4x headroom under fp16 overflow after the x16
scale; the wrapper image with source_precision="fast" (alone, and with precision="fast") against exact; and
video.drive_image_with_video with a fast-source wrapper."""
import ctypes as C
import math
import pathlib
import zlib
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

import conv_plan_cases as CP
from oracle import frames as FR

pytestmark = pytest.mark.gpu
GOLD = pathlib.Path(__file__).parent / "golden"
H1 = "h1"
G = 32
ACC_TOL = 1e-5       # vs float64 on the rounded operands, relative to max(1, scale)
POST_TOL = 5e-5      # GroupNorm post-op, relative to max(1, its largest output)
GUARD = 4096


@dataclass(frozen=True)
class Case:
    Cin: int
    Cout: int
    sp: tuple                  # input (D, H, W)
    k: tuple = (3, 3, 3)       # (kd, kh, kw)
    stride: int = 1            # in H and W
    pad: tuple = None          # (pd, ph, pw); default k // 2
    pool_fold: bool = False    # the (1, 4, 4) stride-2 weight of `3x3 conv -> 2x2 average pool` (ops.fold_poolconv_weight)
    residual: bool = False
    stats: bool = False        # GroupNorm(32) statistics of the output
    post: bool = False         # GroupNorm + ReLU post-op on the convolution's own statistics (nets.ResBlock's first conv)

    @property
    def id(self):
        opts = [o for o in ("pool_fold", "residual", "stats", "post") if getattr(self, o)]
        return (f"{self.Cin}-{self.Cout}-{'x'.join(map(str, self.sp))}-k{''.join(map(str, self.k))}s{self.stride}"
                + "".join("-" + o for o in opts))

    @property
    def padding(self):
        return self.pad if self.pad is not None else tuple(k // 2 for k in self.k)

    @property
    def strides(self):
        return (1, self.stride, self.stride)

    def out_dhw(self):
        return tuple((i + 2 * p - k) // s + 1 for i, k, p, s in zip(self.sp, self.k, self.padding, self.strides))


# plan class at 132 SMs (conv_plan_cases.plan_class(): "<kernel> BN<N tile> <main loop> <finish>", " 3-D" for inputs of
# depth > 1) -> case (the layer each stands for).  The 3-D shapes are the model's with fewer depth slices or rows where that
# keeps the plan class.
CASES = [
    ("h1<32,1> BN96 rr3 none 3-D", Case(96, 96, (16, 64, 64), residual=True, stats=True)),         # VolumeSource, second conv
    ("h1<32,1> BN96 rr3 apply 3-D", Case(96, 96, (16, 64, 64), post=True, stats=True)),            # VolumeSource, first conv
    ("h1<32,1> BN96 tap none 3-D", Case(96, 96, (16, 64, 64), k=(1, 1, 1))),                       # the U-Net head
    ("h1<64,1> BN96 rr3 apply 3-D", Case(192, 96, (8, 64, 64), post=True, stats=True)),            # Cin 192
    ("h1<64,1> BN96 rr3 none 3-D", Case(192, 192, (8, 32, 32), residual=True, stats=True)),
    ("h1<64,1> BN96 tap none 3-D", Case(384, 192, (32, 32, 32), k=(1, 1, 1))),                      # 1^3 skip
    ("h1<64,1> BN128 rr3 apply 3-D", Case(384, 384, (8, 32, 32), post=True, stats=True)),          # Cin 384
    ("h1<64,1> BN128 rr3 none 3-D", Case(512, 512, (16, 16, 16), residual=True, stats=True)),      # Cin 512
    ("h1<64,1> BN128 tap none 3-D", Case(512, 384, (16, 16, 16), k=(1, 1, 1))),
    ("h1<64,1> BN128 tap none", Case(256, 256, (1, 256, 256), k=(1, 4, 4), stride=2, pad=(0, 1, 1), pool_fold=True,
                                     residual=True, stats=True)),                                  # encoder, 256^2
    ("h1<64,1> BN128 tap none", Case(512, 512, (1, 128, 128), k=(1, 4, 4), stride=2, pad=(0, 1, 1), pool_fold=True,
                                     residual=True, stats=True)),
]
# a depth-tiled one-plane tile (td > 1: a box of 2 depth slices x 8 x 8) with split-K, which the shipped models do not reach
DEPTH_CASE = ("h1<32,1> BN96 tap finalize 3-D", Case(96, 96, (4, 8, 8), residual=True, stats=True))


@pytest.fixture(scope="module")
def ops():
    from emoportraits_b200 import ops as o
    return o


def make(c: Case, ops, device="cuda"):
    """seeded fp32 operands of a case (NCDHW): x, w (OIDHW), bias, residual"""
    g = torch.Generator().manual_seed(zlib.crc32(c.id.encode()))
    x = torch.randn((1, c.Cin) + tuple(c.sp), generator=g)
    if c.pool_fold:
        w = ops.fold_poolconv_weight(torch.randn((c.Cout, c.Cin, 3, 3), generator=g) / math.sqrt(c.Cin * 9))[:, :, None]
    else:
        w = torch.randn((c.Cout, c.Cin) + tuple(c.k), generator=g) / math.sqrt(c.Cin * math.prod(c.k))
    b = torch.randn(c.Cout, generator=g)
    res = torch.randn((1, c.Cout) + c.out_dhw(), generator=g) if c.residual else None
    return [t.to(device) if t is not None else None for t in (x, w, b, res)]


def _cl(x):
    return x.permute(0, 2, 3, 4, 1).contiguous()


def _round(x, scale):
    return (x.float() * scale).half().double() / scale


def _gamma_beta(c, device, dtype=torch.float32):
    return (torch.linspace(0.5, 1.5, c.Cout, device=device, dtype=dtype),
            torch.linspace(-0.5, 0.5, c.Cout, device=device, dtype=dtype))


def conv_args(c: Case, ops, x, w, b, res, stats=None):
    """(Split, PackedConvWeight, keyword arguments of ops.conv_igemm / conv_plan) of a case; x may live on the host (planning)"""
    pw = ops.pack_conv_weight(w.cpu(), device=x.device, planes=H1)
    a = ops.split_bf16(_cl(x), H1) if x.is_cuda else ops.Split.empty(_cl(x).shape, x.device, H1)
    kw = dict(stride=c.strides, pad=c.padding, bias=b, residual=_cl(res) if res is not None else None, stats=stats)
    if c.post:
        gamma, beta = _gamma_beta(c, x.device)
        kw["post"] = dict(act=ops.ACT_RELU, planes=H1, want_f32=True, want_split=True,
                          gn=dict(stats=stats, count=math.prod(c.out_dhw()) * c.Cout / G, gamma=gamma, beta=beta))
    return a, pw, kw


def _alloc(shape, dtype, fill=float("nan")):
    """output (filled with `fill`) followed by a NaN guard region: (guard, output view)"""
    n = math.prod(shape)
    buf = torch.full((n + GUARD,), float("nan"), dtype=dtype, device="cuda")
    buf[:n].fill_(fill)
    return buf[n:], buf[:n].view(shape)


def run_guarded(c: Case, ops, a, pw, kw):
    """ops.conv_igemm of the case with every output (the convolution's, its statistics, the post-op's fp32 output and fp16
    plane) written into a buffer followed by a NaN guard; returns ({name: output}, {name: guard})"""
    from emoportraits_b200 import lib as L

    Do, Ho, Wo = c.out_dhw()
    shape = (1, Do, Ho, Wo, c.Cout)
    guards, outs = {}, {}
    guards["conv"], outs["conv"] = _alloc(shape, torch.float32)
    if kw["stats"] is not None:
        guards["stats"], outs["stats"] = _alloc((1, G, 2), torch.float64, fill=0.0)   # the statistics accumulate into zeros
        kw = dict(kw, stats=outs["stats"])
        if "post" in kw:
            kw["post"] = dict(kw["post"], gn=dict(kw["post"]["gn"], stats=outs["stats"]))
    d, _ret, pd, _ = ops._conv_desc(a, pw, kw["stride"], kw["pad"], kw["bias"], kw["residual"], 0, 0, None, False, kw["stats"], G,
                                    outs["conv"], 0, True, False, kw.get("post"))
    if pd is not None:
        guards["post"], outs["post"] = _alloc(shape, torch.float32)
        guards["plane"], outs["plane"] = _alloc(shape, torch.float16)
        pd.out, pd.out_hi = outs["post"].data_ptr(), outs["plane"].data_ptr()
    L.call("emo_conv_igemm", C.byref(d), ops._stream())
    torch.cuda.synchronize()
    return outs, guards


def _ncdhw(t):
    return t.permute(0, 4, 1, 2, 3)


def _check_stats(st, y, scale):
    """the kernel's per-group (sum, sum of squares) of its output against float64 of y (N, C, ...)"""
    r = y.reshape(y.shape[0], G, -1)
    count = r.shape[-1]
    d_mean = (st[..., 0] / count - r.mean(-1)).abs().max().item()
    msq = (r * r).mean(-1)
    d_msq = ((st[..., 1] / count - msq).abs() / msq).max().item()
    assert d_mean < 1e-6 * scale and d_msq < 1e-5, (d_mean, d_msq)
    return f" stats: mean {d_mean:.1e}, mean-square {d_msq:.1e} (rel)"


def check_case(ops, want, c, depth_tiled=False):
    x, w, b, res = make(c, ops)
    st = torch.zeros((1, G, 2), dtype=torch.float64, device="cuda") if c.stats else None
    a, pw, kw = conv_args(c, ops, x, w, b, res, st)
    info = ops.conv_plan(a, pw, **kw)
    assert info.NP == 1 and info.fp16 == 1
    assert (info.td > 1) == depth_tiled, info.td
    if torch.cuda.get_device_properties(0).multi_processor_count == 132:
        assert CP.plan_class(info, c.sp[0]) == want, (CP.plan_class(info, c.sp[0]), want)
    outs, guards = run_guarded(c, ops, a, pw, kw)
    for name, g in guards.items():
        assert torch.isnan(g.float()).all(), f"{name}: write past the end of the output"
    ck = dict(stride=c.strides, padding=c.padding)
    y_r = F.conv3d(_round(x, ops.F16_ACT_SCALE), _round(w, ops.F16_W_SCALE), **ck)
    y_x = F.conv3d(x.double(), w.double(), **ck)
    opb = F.conv3d(x.double().abs(), w.double().abs(), **ck) * 2.0 ** -10
    extra = b.double().view(1, -1, 1, 1, 1) + (res.double() if res is not None else 0.0)
    y_r, y_x = y_r + extra, y_x + extra
    scale = max(y_r.abs().max().item(), 1.0)
    out = _ncdhw(outs["conv"]).double()
    assert not torch.isnan(out).any(), "output not fully written"
    e_acc = (out - y_r).abs().max().item()
    excess = ((out - y_x).abs() - opb).max().item()
    msg = (f"\n[{want} {c.id}] td {info.td} ksplit {info.ksplit}: vs rounded operands {e_acc:.2e} ({e_acc / scale:.1e} of scale "
           f"{scale:.1f}); vs fp32 operands {(out - y_x).abs().max().item():.2e}, excess over the operand bound {excess:.1e}")
    assert e_acc < ACC_TOL * scale, (e_acc, scale)
    assert excess < ACC_TOL * scale, excess
    if c.stats:
        msg += _check_stats(outs["stats"], y_r, scale)
    if c.post:
        gamma, beta = _gamma_beta(c, "cuda", torch.float64)
        pref = torch.relu(F.group_norm(y_r, G, gamma, beta, 1e-5))
        bound = POST_TOL * max(1.0, pref.abs().max().item())
        pout, plane = _ncdhw(outs["post"]).double(), _ncdhw(outs["plane"]).double() / ops.F16_ACT_SCALE
        assert not torch.isnan(pout).any() and not torch.isnan(plane).any(), "post-op output not fully written"
        pe = (pout - pref).abs().max().item()
        ple = ((plane - pref).abs() - 2.0 ** -11 * pref.abs()).max().item()
        msg += f"; post-op {pe:.2e}, its fp16 plane's excess over fp16 rounding {ple:.2e}"
        assert pe < bound, pe
        assert ple < bound, ple
    print(msg)


@pytest.mark.parametrize("want,c", CASES, ids=[f"{w}-{c.id}" for w, c in CASES])
def test_one_plane_source_conv_against_float64(ops, want, c):
    check_case(ops, want, c)


def test_one_plane_depth_tiled_conv_against_float64(ops):
    check_case(ops, *DEPTH_CASE, depth_tiled=True)


# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [256, 512])
def test_stem_with_statistics_against_float64_and_conv_direct(ops, S):
    """the local encoder's stem in fast mode (stem_pack + 7x1 implicit GEMM with GroupNorm statistics) on the resized RGB of a
    frame: vs float64 F.conv2d (7x7, pad 3) on the rounded operands, vs conv_direct within the operand bound, and its
    statistics vs float64 (and vs conv_direct's)"""
    from emoportraits_b200 import nets
    from emoportraits_b200.checkpoint import synthetic_state_dict
    from emoportraits_b200.config import shipped_config

    sd = synthetic_state_dict(shipped_config(S), 0)
    w_dir, b = nets.stem_weight(sd, f"local_encoder_nw.from_rgb_{S}px", "cuda")
    img = FR.frame(S, 21, "noise").cuda()
    x4 = ops.resize_bilinear(img, (S, S))
    Co = w_dir.shape[-1]
    guard, out = _alloc((1, 1, S, S, Co), torch.float32)
    sguard, st = _alloc((1, G, 2), torch.float64, fill=0.0)
    got = ops.conv_igemm(ops.stem_pack(x4), ops.pack_stem_weight(w_dir.cpu(), device="cuda"), pad=(0, 3, 0), bias=b, stats=st,
                         out=out)
    torch.cuda.synchronize()
    assert torch.isnan(guard).all() and torch.isnan(sguard).all() and not torch.isnan(got).any()
    st_direct = torch.zeros((1, G, 2), dtype=torch.float64, device="cuda")
    direct = ops.conv_direct(x4, w_dir, 1, 3, b, stats=st_direct)
    x = x4[:, 0, :, :, :3].permute(0, 3, 1, 2).double()
    w = w_dir[:, :, :3].permute(3, 2, 0, 1).double()               # (7, 7, 4, Co) -> (Co, 3, 7, 7)
    bb = b.double().view(1, -1, 1, 1)
    y_r = F.conv2d(_round(x, ops.F16_ACT_SCALE), _round(w, ops.F16_W_SCALE), padding=3) + bb
    opb = F.conv2d(x.abs(), w.abs(), padding=3) * 2.0 ** -10
    scale = max(y_r.abs().max().item(), 1.0)
    g = got[:, 0].permute(0, 3, 1, 2).double()
    e_acc = (g - y_r).abs().max().item()
    excess = ((g - direct[:, 0].permute(0, 3, 1, 2).double()).abs() - opb).max().item()
    msg = (f"\n[stem {S}^2 with statistics] vs rounded operands {e_acc:.2e} ({e_acc / scale:.1e} of scale {scale:.2f}); vs "
           f"conv_direct {(got - direct).abs().max().item():.2e}, excess over the operand bound {excess:.1e};")
    assert e_acc < ACC_TOL * scale, e_acc
    assert excess < ACC_TOL * scale, excess
    msg += _check_stats(st, y_r, scale)
    # against the exact mode's statistics: a group mean moves by at most the largest operand bound
    count = S * S * Co / G
    d_direct = (st[..., 0] / count - st_direct[..., 0] / count).abs().max().item()
    msg += f"; group mean vs conv_direct's {d_direct:.1e}"
    assert d_direct < opb.max().item() + ACC_TOL * scale, d_direct
    print(msg)


# ------------------------------------------------------------------------------------------------------------------
# model level.  Bounds from tools/decoder_precision_emulation.py --source (synthetic seed-0 weights, oracle frames 21 -> 22,
# smooth and noise; DESIGN.md section 2 has the table).  Row "source h1": target_latent_volume max-abs 2.5e-3 / 3.0e-3 at
# 256^2 / 512^2 (of a largest value 2.4), image PSNR >= 70.9 / 68.9 dB, every uint8 pixel within one level.  Row "both fast"
# (precision="fast" too): image max-abs 3.0e-3 / 4.1e-3, PSNR >= 67.8 / 65.5 dB, uint8 pixels within one level at 256^2 and
# up to two at 512^2 (4.1e-3 is more than one level, 1/255).  Bounds: about 3x the emulated latent error, and ~10 dB (3x the
# RMS error) under the emulated PSNR.
LATENT_BOUND = 1e-2
PSNR_BOUND = 60.0
BOTH_LEVELS = 2
BOTH_PSNR_BOUND = 55.0
MAX_ACTIVATION = 65504.0 / 16 / 4


@pytest.fixture(scope="module", params=[256, 512])
def src_ctx(request):
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import Model

    size = request.param
    cfg = shipped_config(size)
    sd, hsd = synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0)
    return dict(size=size, cfg=cfg, sd=sd, hsd=hsd, Model=Model)


UNSWITCHED = ("idt_embed", "pred_source_theta", "pred_source_pose_embed", "source_xy_warp_resize")


def test_fast_source_pass_against_exact(ops, src_ctx, monkeypatch):
    Model, cfg = src_ctx["Model"], src_ctx["cfg"]
    exact = Model(cfg, src_ctx["sd"], src_ctx["hsd"], "cuda")
    fast = Model(cfg, src_ctx["sd"], src_ctx["hsd"], "cuda", precision=dict(Model.SOURCE_FAST))
    assert fast.local_encoder_nw.stem_h1 is not None and exact.local_encoder_nw.stem_h1 is None
    src = FR.frame(src_ctx["size"], 21, "noise").cuda()
    st_e = exact.source_pass(src)
    # the largest activation any one-plane convolution reads (its plane holds fp16(16 x), saturating at 65504)
    seen = []
    conv = ops.conv_igemm

    def watch(a, *args, **kw):
        if a.lo is None:
            seen.append(a.hi.float().abs().max().item() / a.scale)
        return conv(a, *args, **kw)

    monkeypatch.setattr(ops, "conv_igemm", watch)
    st_f = fast.source_pass(src)
    monkeypatch.setattr(ops, "conv_igemm", conv)
    st_f2 = fast.source_pass(src)
    torch.cuda.synchronize()
    for name in UNSWITCHED:
        assert torch.equal(getattr(st_f, name), getattr(st_e, name)), name
    for name in ("source_latent_volume", "target_latent_volume_1", "target_latent_volume"):
        assert torch.equal(getattr(st_f, name), getattr(st_f2, name)), name               # two runs bit-identical
    tlv_e, tlv_f = st_e.target_latent_volume, st_f.target_latent_volume
    assert not torch.isnan(tlv_f).any()
    e_tlv = (tlv_f - tlv_e).abs().max().item()
    e_slv = (st_f.source_latent_volume - st_e.source_latent_volume).abs().max().item()
    n_one = len(seen)
    print(f"\n[fast source pass @{src_ctx['size']}] target_latent_volume max-abs {e_tlv:.2e} (of max {tlv_e.abs().max().item():.2f}), "
          f"source_latent_volume max-abs {e_slv:.2e}; largest |activation| into a one-plane conv {max(seen):.2f} over {n_one} "
          f"convolutions (bound {MAX_ACTIVATION:.0f})")
    assert n_one > 0 and e_tlv < LATENT_BOUND
    assert max(seen) < MAX_ACTIVATION


def _wrapper(tmp_path, ctx, **kw):
    from emoportraits_b200.infer import InferenceWrapper

    exp = tmp_path / "logs" / "exp" / "checkpoints"
    if not exp.exists():
        exp.mkdir(parents=True)
        (tmp_path / "logs" / "exp" / "args.txt").write_text((GOLD / f"args_{ctx['size']}.txt").read_text())
        torch.save(ctx["sd"], exp / "000_model.pth")
    return InferenceWrapper(experiment_name="exp", model_file_name="000_model.pth", project_dir=str(tmp_path), folder="logs",
                            print_params=False, head_pose_state_dict=ctx["hsd"], **kw)


def _u8(pils):
    import numpy as np

    return torch.from_numpy(np.stack([np.asarray(p) for p in pils]).astype("int32"))


def _psnr(a, b):
    return [10 * math.log10(1.0 / ((a[i] - b[i]) ** 2).mean().item()) for i in range(a.shape[0])]


def test_fast_source_wrapper_against_exact(src_ctx, tmp_path):
    """photo-to-photo (forward(source, driver)) and a list of driver frames, source_precision="fast" against "exact", alone and
    together with precision="fast"; the second call is bit-identical to the first"""
    from emoportraits_b200 import ops

    size = src_ctx["size"]
    exact = _wrapper(tmp_path, src_ctx)
    fast = _wrapper(tmp_path, src_ctx, source_precision="fast")
    both = _wrapper(tmp_path, src_ctx, precision="fast", source_precision="fast")
    assert exact.source_precision == "exact" and fast.source_precision == "fast" and fast.precision == "exact"
    assert fast.model.precision["unet3d"] == ops.H1 and fast.model.precision["decoder"] == 2
    assert both.model.precision["decoder"] == ops.H1 and both.model.precision["warp"] == ops.H2
    src = FR.pil(size, 21, "smooth")
    drv = [FR.pil(size, 60 + i, "smooth") for i in range(3)]
    fw = dict(crop=False, mix=True, mix_old=False)
    pil_e, img_e = exact.forward(src, drv, **fw)
    pil_f, img_f = fast.forward(src, drv, **fw)
    pil_f2, img_f2 = fast.forward(src, drv, **fw)
    pil_b, img_b = both.forward(src, drv, **fw)
    one_e, _ = exact.forward(src, drv[0], **fw)                      # photo to photo: one source pass + one driver frame
    one_f, _ = fast.forward(src, drv[0], **fw)
    d_u8 = (_u8(pil_f) - _u8(pil_e)).abs()
    d_one = (_u8(one_f) - _u8(one_e)).abs()
    d_both = (_u8(pil_b) - _u8(pil_e)).abs()
    psnr, psnr_b = _psnr(img_f, img_e), _psnr(img_b, img_e)
    print(f"\n[source_precision=fast vs exact @{size}] uint8 max {d_u8.max().item()} level(s), "
          f"{100 * (d_u8 > 0).float().mean().item():.2f} % of pixels moved, image max-abs {(img_f - img_e).abs().max().item():.1e}, "
          f"PSNR min {min(psnr):.1f} dB; photo-to-photo max {d_one.max().item()} level(s)\n"
          f"[precision=fast + source_precision=fast vs exact @{size}] uint8 max {d_both.max().item()} level(s), "
          f"{100 * (d_both > 0).float().mean().item():.2f} % moved, PSNR min {min(psnr_b):.1f} dB")
    assert d_u8.max().item() <= 1 and d_one.max().item() <= 1
    assert min(psnr) >= PSNR_BOUND
    assert torch.equal(_u8(pil_f), _u8(pil_f2)) and torch.equal(img_f, img_f2)     # two runs bit-identical
    assert d_both.max().item() <= BOTH_LEVELS
    assert min(psnr_b) >= BOTH_PSNR_BOUND


def test_drive_image_with_video_runs_with_a_fast_source_wrapper(tmp_path):
    """video.drive_image_with_video with a source_precision="fast" wrapper == that wrapper's source pass and driver frames"""
    from emoportraits_b200 import video
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config

    size = 256
    cfg = shipped_config(size)
    ctx = dict(size=size, sd=synthetic_state_dict(cfg, 0), hsd=synthetic_head_pose_state_dict(0))
    w = _wrapper(tmp_path, ctx, source_precision="fast")
    src = FR.pil(size, 41, "smooth")
    frames = [FR.pil(size, 50 + i, "smooth") for i in range(5)]
    outs, _, _ = video.drive_image_with_video(w, src, frames, chunk=3)
    tlv = w.target_latent_volume.clone()
    want, _ = w.forward(src, frames, crop=False, smooth_pose=False, target_theta=True, mix=True, mix_old=False)
    assert len(outs) == 5 and torch.equal(tlv, w.target_latent_volume)
    assert torch.equal(_u8(outs), _u8(want))
