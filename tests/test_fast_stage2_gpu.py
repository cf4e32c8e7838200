"""GPU tests of stage 2's fast mode (stage2.Stage2Model(precision="fast"): every convolution on one fp16 operand plane, ops.H1,
and the 7x7 RGB stem as a 7x1 implicit GEMM over ops.stem_pack's 32 channels).

Op level, one case per one-plane plan class that fast-mode stage 2 reaches and tests/test_fast_decoder_gpu.py does not sweep
(tests/test_fast_stage2_cpu.py checks that the two tables cover every stage-2 convolution at 512^2 and 1024^2), every output
written into NaN with a NaN guard region after it:
  * within 1e-5 of the scale of float64 on the ROUNDED operands, fp16(x * 16) / 16 and fp16(w * 256) / 256;
  * within the one-plane operand bound 2^-10 conv(|x|, |w|) (+ 1e-5 of the scale) of float64 on the fp32 operands;
  * the BatchNorm-affine post-op in fp32 and its one fp16 plane within fp16 rounding of the float64 post-op.
The stem: emo_stem_pack's plane is bit-equal to a host-built fp16 im2col; the stem convolution matches float64 F.conv2d on the
rounded operands within 1e-5 of the scale and conv_direct (the exact mode's stem) within the operand bound.
Model level (synthetic seed-0 weights, tools/decoder_precision_emulation.py --stage2 gives the bounds): the latent and `add`
against the reference fixtures, every ffhq uint8 pixel within one level; the wrapper fast against exact (uint8 within one
level, PSNR bound, two runs bit-identical); video.drive_image_with_video with a fast stage-2 wrapper; and the largest
activation any one-plane convolution reads, with 4x headroom under fp16 overflow after the x16 scale."""
import ctypes as C
import math
import pathlib
import zlib
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

from oracle import frames as FR

pytestmark = pytest.mark.gpu
GOLD = pathlib.Path(__file__).parent / "golden"
H1 = "h1"
ACC_TOL = 1e-5       # vs float64 on the rounded operands, relative to max(1, scale)
GUARD = 4096
RELU, TANH = 1, 3


@dataclass(frozen=True)
class Case:
    Cin: int
    Cout: int
    sp: tuple                  # input (H, W)
    k: tuple = (3, 3)          # (kh, kw)
    stride: int = 1
    pad: tuple = None          # (ph, pw); default k // 2
    N: int = 1
    pool_fold: bool = False    # the 4x4 stride-2 weight of `3x3 conv -> 2x2 average pool` (ops.fold_poolconv_weight)
    residual: bool = False
    post: bool = False         # eval-BatchNorm affine + ReLU post-op (nets.Norm.apply_args of a folded BatchNorm)
    act: int = 0
    out_nchw: bool = False

    @property
    def id(self):
        opts = [o for o in ("pool_fold", "residual", "post", "out_nchw") if getattr(self, o)] + ([f"act{self.act}"] if self.act else [])
        return f"N{self.N}-{self.Cin}-{self.Cout}-{self.sp[0]}x{self.sp[1]}-k{self.k[0]}{self.k[1]}s{self.stride}" + "".join("-" + o for o in opts)

    @property
    def padding(self):
        return self.pad if self.pad is not None else (self.k[0] // 2, self.k[1] // 2)

    def out_hw(self):
        return tuple((i + 2 * p - k) // self.stride + 1 for i, k, p in zip(self.sp, self.k, self.padding))


# plan class at 132 SMs -> case (the stage-2 layer each stands for)
CASES = [
    ("h1<32,1> BN128 rr3 none", Case(32, 128, (96, 96), k=(7, 1), pad=(3, 0))),                        # the stem, 7x1 over stem_pack
    ("h1<64,1> BN128 tap none", Case(128, 128, (192, 192), k=(4, 4), stride=2, pad=(1, 1), pool_fold=True, residual=True)),
    ("h1<64,1> BN128 rr3 apply", Case(128, 128, (128, 128), post=True)),                                 # BatchNorm post, no stats
    ("h1<64,1> BN64 rr3 apply", Case(128, 64, (96, 96), post=True)),
    ("h1<64,1> BN32 rr3 apply", Case(64, 32, (96, 96), post=True)),
    ("h1<64,1> BN64 rr3 none", Case(64, 64, (96, 96), residual=True)),
    ("h1<64,1> BN64 tap none", Case(128, 64, (96, 96), k=(1, 1))),
    ("h1<64,1> BN32 tap none", Case(64, 32, (96, 96), k=(1, 1))),
    ("h1<32,1> BN32 rr3 none", Case(32, 32, (96, 96), residual=True)),
    ("h1<32,1> BN16 tap none", Case(32, 3, (64, 64), k=(1, 1), act=TANH, out_nchw=True, N=2)),         # the 32 -> 3 tanh head
]


@pytest.fixture(scope="module")
def ops():
    from emoportraits_b200 import ops as o
    return o


def make(c: Case, ops, device="cuda"):
    """seeded fp32 operands of a case (NCHW): x, w (OIHW), bias, residual, BatchNorm affine (A, B)"""
    g = torch.Generator().manual_seed(zlib.crc32(c.id.encode()))
    x = torch.randn((c.N, c.Cin) + tuple(c.sp), generator=g)
    if c.pool_fold:
        w = ops.fold_poolconv_weight(torch.randn((c.Cout, c.Cin, 3, 3), generator=g) / math.sqrt(c.Cin * 9))
    else:
        w = torch.randn((c.Cout, c.Cin) + tuple(c.k), generator=g) / math.sqrt(c.Cin * c.k[0] * c.k[1])
    b = torch.randn(c.Cout, generator=g)
    res = torch.randn((c.N, c.Cout) + c.out_hw(), generator=g) if c.residual else None
    A = (torch.rand(c.Cout, generator=g) + 0.5) if c.post else None
    B = torch.randn(c.Cout, generator=g) * 0.5 if c.post else None
    return [t.to(device) if t is not None else None for t in (x, w, b, res, A, B)]


def _round(x, scale):
    return (x.float() * scale).half().double() / scale


def _cl(x):
    return x.permute(0, 2, 3, 1).contiguous()[:, None]


def _alloc(shape, dtype):
    """NaN-filled output followed by a NaN guard region: (guard, output view)"""
    n = math.prod(shape)
    buf = torch.full((n + GUARD,), float("nan"), dtype=dtype, device="cuda")
    return buf[n:], buf[:n].view(shape)


def _plan_class(info):
    from emoportraits_b200 import lib as L

    loop = f"rr{info.sa}" if info.yreuse else "tap"
    return f"{L.conv_kernel_name(info.kernel)} BN{info.BN} {loop} {L.CONV_FINISH[info.finish]}"


def conv_args(c: Case, ops, x, w, b, res, A, B):
    """(Split, PackedConvWeight, keyword arguments of ops.conv_igemm / conv_plan) of a case; x may live on the host (planning)"""
    pw = ops.pack_conv_weight(w.cpu(), device=x.device, planes=H1)
    a = ops.split_bf16(_cl(x), H1) if x.is_cuda else ops.Split.empty(_cl(x).shape, x.device, H1)
    kw = dict(stride=(1, c.stride, c.stride), pad=(0,) + tuple(c.padding), bias=b, residual=_cl(res) if res is not None else None,
              act=c.act, out_nchw=c.out_nchw)
    if c.post:
        kw["post"] = dict(A=A[None].contiguous(), B=B[None].contiguous(), per_sample=False, act=ops.ACT_RELU, planes=H1,
                          want_f32=True, want_split=True)
    return a, pw, kw


def run_guarded(c: Case, ops, a, pw, kw):
    """ops.conv_igemm of the case with every output (the convolution's, and the post-op's fp32 output and fp16 plane) written
    into a NaN buffer followed by a NaN guard; returns ({name: output}, {name: guard})"""
    from emoportraits_b200 import lib as L

    Ho, Wo = c.out_hw()
    shape = (c.N, c.Cout, 1, Ho, Wo) if c.out_nchw else (c.N, 1, Ho, Wo, c.Cout)
    guards, outs = {}, {}
    guards["conv"], outs["conv"] = _alloc(shape, torch.float32)
    d, _ret, pd, _ = ops._conv_desc(a, pw, kw["stride"], kw["pad"], kw["bias"], kw["residual"], 0, kw["act"], None, kw["out_nchw"],
                                    None, 32, outs["conv"], 0, True, False, kw.get("post"))
    if pd is not None:
        guards["post"], outs["post"] = _alloc((c.N, 1, Ho, Wo, c.Cout), torch.float32)
        guards["plane"], outs["plane"] = _alloc((c.N, 1, Ho, Wo, c.Cout), torch.float16)
        pd.out, pd.out_hi = outs["post"].data_ptr(), outs["plane"].data_ptr()
    L.call("emo_conv_igemm", C.byref(d), ops._stream())
    torch.cuda.synchronize()
    return outs, guards


def _nchw(c, t):
    return t[:, :, 0] if c.out_nchw else t[:, 0].permute(0, 3, 1, 2)


@pytest.mark.parametrize("want,c", CASES, ids=[w for w, _ in CASES])
def test_one_plane_stage2_conv_against_float64(ops, want, c):
    x, w, b, res, A, B = make(c, ops)
    a, pw, kw = conv_args(c, ops, x, w, b, res, A, B)
    info = ops.conv_plan(a, pw, **kw)
    assert info.NP == 1 and info.fp16 == 1
    if torch.cuda.get_device_properties(0).multi_processor_count == 132:
        assert _plan_class(info) == want, (_plan_class(info), want)
    outs, guards = run_guarded(c, ops, a, pw, kw)
    for name, g in guards.items():
        assert torch.isnan(g.float()).all(), f"{name}: write past the end of the output"
    ck = dict(stride=c.stride, padding=c.padding)
    y_r = F.conv2d(_round(x, ops.F16_ACT_SCALE), _round(w, ops.F16_W_SCALE), **ck)
    y_x = F.conv2d(x.double(), w.double(), **ck)
    opb = F.conv2d(x.double().abs(), w.double().abs(), **ck) * 2.0 ** -10
    extra = b.double().view(1, -1, 1, 1) + (res.double() if res is not None else 0.0)
    y_r, y_x = y_r + extra, y_x + extra
    scale = max(y_r.abs().max().item(), 1.0)
    if c.act == TANH:
        y_r, y_x = torch.tanh(y_r), torch.tanh(y_x)     # tanh is 1-Lipschitz: the bounds carry over
    out = _nchw(c, outs["conv"]).double()
    assert not torch.isnan(out).any(), "output not fully written"
    e_acc = (out - y_r).abs().max().item()
    excess = ((out - y_x).abs() - opb).max().item()
    msg = (f"\n[{want}] ksplit {info.ksplit}: vs rounded operands {e_acc:.2e} ({e_acc / scale:.1e} of scale {scale:.1f}); "
           f"vs fp32 operands {(out - y_x).abs().max().item():.2e}, excess over the operand bound {excess:.1e}")
    assert e_acc < ACC_TOL * scale, (e_acc, scale)
    assert excess < ACC_TOL * scale, excess
    if c.post:
        pref = torch.relu(y_r * A.double().view(1, -1, 1, 1) + B.double().view(1, -1, 1, 1))
        bound = ACC_TOL * scale * max(1.0, A.abs().max().item())
        pout, plane = _nchw(c, outs["post"]).double(), _nchw(c, outs["plane"]).double() / ops.F16_ACT_SCALE
        assert not torch.isnan(pout).any() and not torch.isnan(plane).any(), "post-op output not fully written"
        pe = (pout - pref).abs().max().item()
        ple = ((plane - pref).abs() - 2.0 ** -11 * pref.abs()).max().item()
        msg += f"; post-op {pe:.2e}, its fp16 plane's excess over fp16 rounding {ple:.2e}"
        assert pe < bound, pe
        assert ple < bound, ple
    print(msg)


# ------------------------------------------------------------------------------------------------------------------
def _stem_im2col(x4, scale):
    """host fp16 im2col of emo_stem_pack: x4 (N,1,H,W,4) -> (N,1,H,W,32), channel kx*4 + c = fp16(scale x[.., w + kx - 3, c])"""
    N, _, H, W, _ = x4.shape
    xp = F.pad(x4, (0, 0, 3, 3))                                   # zero columns outside the image
    cols = [xp[:, :, :, kx:kx + W] for kx in range(7)] + [torch.zeros_like(x4)]
    return (torch.cat(cols, -1) * scale).half()


@pytest.mark.parametrize("N,H,W", [(1, 64, 96), (2, 37, 53), (1, 3, 2)])
def test_stem_pack_bits(ops, N, H, W):
    torch.manual_seed(3)
    x4 = torch.randn(N, 1, H, W, 4, device="cuda")
    sp = ops.stem_pack(x4)
    assert sp.lo is None and sp.f16 and sp.scale == ops.F16_ACT_SCALE and sp.shape == (N, 1, H, W, 32)
    want = _stem_im2col(x4, ops.F16_ACT_SCALE)
    assert torch.equal(sp.hi.view(torch.int16), want.view(torch.int16))
    # the kernel writes exactly N*H*W*32 halves: a NaN guard after the plane stays NaN
    guard, out = _alloc((N, 1, H, W, 32), torch.float16)
    from emoportraits_b200 import lib as L
    L.call("emo_stem_pack", x4.data_ptr(), N, H, W, 4, C.c_float(ops.F16_ACT_SCALE), out.data_ptr(), ops._stream())
    torch.cuda.synchronize()
    assert torch.isnan(guard.float()).all() and torch.equal(out.view(torch.int16), want.view(torch.int16))


@pytest.mark.parametrize("N,S", [(1, 128), (2, 96)])
def test_stem_conv_against_float64_and_conv_direct(ops, N, S):
    """the stem of Stage2Model(precision="fast") on resized RGB: vs float64 F.conv2d (7x7, pad 3) on the rounded operands and
    vs conv_direct, the exact mode's stem, within the operand bound"""
    from emoportraits_b200 import nets
    from emoportraits_b200.stage2 import Stage2Config, synthetic_state_dict_s2

    cfg = Stage2Config(output_size=512)
    sd = synthetic_state_dict_s2(cfg, 0)
    w_dir, b = nets.stem_weight(sd, "local_encoder.from_rgb_512px", "cuda")
    x4 = ops.resize_bilinear(FR.frame(256, 21, "smooth").repeat(N, 1, 1, 1).cuda() * torch.linspace(0.5, 1, N, device="cuda").view(N, 1, 1, 1),
                             (S, S))
    guard, out = _alloc((N, 1, S, S, w_dir.shape[-1]), torch.float32)
    got = ops.conv_igemm(ops.stem_pack(x4), ops.pack_stem_weight(w_dir.cpu(), device="cuda"), pad=(0, 3, 0), bias=b, out=out)
    torch.cuda.synchronize()
    assert torch.isnan(guard).all() and not torch.isnan(got).any()
    direct = ops.conv_direct(x4, w_dir, 1, 3, b)
    x = x4[:, 0, :, :, :3].permute(0, 3, 1, 2).double()
    w = w_dir[:, :, :3].permute(3, 2, 0, 1).double()               # (7, 7, 4, Co) -> (Co, 3, 7, 7)
    bb = b.double().view(1, -1, 1, 1)
    y_r = F.conv2d(_round(x, ops.F16_ACT_SCALE), _round(w, ops.F16_W_SCALE), padding=3) + bb
    opb = F.conv2d(x.abs(), w.abs(), padding=3) * 2.0 ** -10
    scale = max(y_r.abs().max().item(), 1.0)
    g = got[:, 0].permute(0, 3, 1, 2).double()
    e_acc = (g - y_r).abs().max().item()
    excess = ((g - direct[:, 0].permute(0, 3, 1, 2).double()).abs() - opb).max().item()
    print(f"\n[stem {N}x{S}^2] vs rounded operands {e_acc:.2e} ({e_acc / scale:.1e} of scale {scale:.2f}); vs conv_direct "
          f"{(got - direct).abs().max().item():.2e}, excess over the operand bound {excess:.1e}")
    assert e_acc < ACC_TOL * scale, e_acc
    assert excess < ACC_TOL * scale, excess


# ------------------------------------------------------------------------------------------------------------------
# model level.  Bounds from tools/decoder_precision_emulation.py --stage2, row "h1, stem h1 too" (synthetic seed-0 weights;
# 512^2, smooth / noise frame): latent max-abs 1.6e-4 / 1.3e-4, add max-abs 9.2e-5 / 8.5e-5, ffhq PSNR 94.3 / 94.7 dB against
# fp32.  Bounds: about 3x the errors, and 3x the RMS error (~10 dB) for the PSNR.  DESIGN.md section 2 has the measured values.
LATENT_BOUND = 5e-4
ADD_BOUND = 3e-4
PSNR_BOUND = 85.0
MAX_ACTIVATION = 65504.0 / 16 / 4


def _sub_err(got, ref_pair):
    vals, stride = ref_pair
    return (got.detach().float().cpu().reshape(-1)[::stride] - vals).abs().max().item()


def _inputs(gold):
    return torch.cat([FR.frame(gold["input_size"], s, "smooth") for s in gold["seeds"]])


@pytest.fixture(scope="module", params=["s2_512_b1.pt", "s2_1024_b4.pt"])
def s2_ctx(request):
    from emoportraits_b200.stage2 import Stage2Config, synthetic_state_dict_s2

    gold = torch.load(GOLD / request.param, weights_only=False)
    cfg = Stage2Config(output_size=gold["output_size"])
    return dict(name=request.param, gold=gold, cfg=cfg, sd=synthetic_state_dict_s2(cfg, 0))


def test_fast_stage2_against_reference_fixture(ops, s2_ctx, monkeypatch):
    from emoportraits_b200.stage2 import Stage2Model

    gold, cfg = s2_ctx["gold"], s2_ctx["cfg"]
    model = Stage2Model(cfg, s2_ctx["sd"], "cuda", precision="fast")
    assert model.planes == H1 and model.stem_h1 is not None
    img = _inputs(gold).cuda()
    # the largest activation any one-plane convolution reads (its plane holds fp16(16 x), saturating at 65000)
    seen = []
    conv = ops.conv_igemm

    def watch(a, *args, **kw):
        assert a.lo is None and a.f16, "fast mode: every convolution reads one fp16 plane"
        seen.append(a.hi.float().abs().max().item() / a.scale)
        return conv(a, *args, **kw)

    monkeypatch.setattr(ops, "conv_igemm", watch)
    x4 = ops.resize_bilinear(img, (cfg.output_size, cfg.output_size))
    vol = model.local_encoder(x4)
    e_vol = _sub_err(vol[:, 0].permute(0, 3, 1, 2).contiguous(), gold["vol"])
    resized, add, ffhq = model.forward(img)
    monkeypatch.setattr(ops, "conv_igemm", conv)
    torch.cuda.synchronize()
    assert not torch.isnan(add).any()
    e_add = _sub_err(add, gold["add"])
    e_img = _sub_err((ffhq * 255).floor().clamp(0, 255).permute(0, 2, 3, 1).contiguous(), gold["ffhq_uint8"])
    print(f"\n[fast stage 2 vs reference golden {s2_ctx['name']}] latent {e_vol:.2e} add {e_add:.2e} ffhq(uint8 steps) {e_img:.0f}; "
          f"largest |activation| into a one-plane conv {max(seen):.2f} over {len(seen)} convolutions (bound {MAX_ACTIVATION:.0f})")
    assert e_vol < LATENT_BOUND and e_add < ADD_BOUND and e_img <= 1.0
    assert max(seen) < MAX_ACTIVATION


def _wrapper(tmp_path, s2_ctx, precision):
    from emoportraits_b200.stage2 import InferenceWrapper

    d = tmp_path / "logs_s2" / "exp" / "checkpoints"
    if not d.exists():
        d.mkdir(parents=True)
        (tmp_path / "logs_s2" / "exp" / "args.txt").write_text((GOLD / f"args_s2_{s2_ctx['cfg'].output_size}.txt").read_text())
        torch.save(s2_ctx["sd"], d / "m.pth")
    return InferenceWrapper(experiment_name="exp", model_file_name="m.pth", project_dir=str(tmp_path), precision=precision)


def _u8(pils):
    import numpy as np

    return torch.from_numpy(np.stack([np.asarray(p) for p in pils]).astype("int32"))


def test_fast_stage2_wrapper_against_exact(s2_ctx, tmp_path):
    exact, fast = _wrapper(tmp_path, s2_ctx, "exact"), _wrapper(tmp_path, s2_ctx, "fast")
    assert exact.model_two.planes == 2 and fast.model_two.planes == H1 and fast.precision == "fast"
    img = _inputs(s2_ctx["gold"]).cuda()
    _, _, pil_e, _ = exact.forward(img)
    _, _, pil_f, _ = fast.forward(img)
    _, _, pil_f2, _ = fast.forward(img)
    d_u8 = (_u8(pil_f) - _u8(pil_e)).abs()
    _, _, ffhq_e = exact.model_two.forward(img)
    _, _, ffhq_f = fast.model_two.forward(img)
    _, _, ffhq_f2 = fast.model_two.forward(img)
    psnr = [10 * math.log10(1.0 / ((ffhq_f[i] - ffhq_e[i]) ** 2).mean().item()) for i in range(img.shape[0])]
    print(f"\n[fast vs exact stage-2 wrapper {s2_ctx['name']}] uint8 max {d_u8.max().item()} level(s), "
          f"{100 * (d_u8 > 0).float().mean().item():.2f} % of pixels changed; ffhq max-abs {(ffhq_f - ffhq_e).abs().max().item():.1e}, "
          f"PSNR min {min(psnr):.1f} dB")
    assert d_u8.max().item() <= 1
    assert min(psnr) >= PSNR_BOUND
    assert torch.equal(_u8(pil_f), _u8(pil_f2)) and torch.equal(ffhq_f, ffhq_f2)     # two runs bit-identical


def test_drive_image_with_video_runs_stage2_fast(tmp_path):
    """video.drive_image_with_video with a fast stage-2 wrapper (512^2) == that wrapper called on the same chunks"""
    from emoportraits_b200 import video
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import InferenceWrapper
    from emoportraits_b200.stage2 import Stage2Config, synthetic_state_dict_s2

    size = 256
    cfg = shipped_config(size)
    w1 = InferenceWrapper(experiment_name="x", project_dir=str(tmp_path), args_path=GOLD / f"args_{size}.txt",
                          state_dict=synthetic_state_dict(cfg, 0), head_pose_state_dict=synthetic_head_pose_state_dict(0),
                          print_params=False)
    cfg2 = Stage2Config(output_size=512)
    w2 = _wrapper(tmp_path, dict(cfg=cfg2, sd=synthetic_state_dict_s2(cfg2, 0)), "fast")
    chunks = []
    fwd = w2.forward

    def record(img, *a, **k):
        chunks.append(img.clone())
        return fwd(img, *a, **k)

    w2.forward = record
    outs, _, _ = video.drive_image_with_video(w1, FR.pil(size, 41, "smooth"), [FR.pil(size, 50 + i, "smooth") for i in range(5)],
                                              inferer_s2=w2, chunk=3)
    w2.forward = fwd
    assert [c.shape[0] for c in chunks] == [3, 2] and len(outs) == 5
    want = [p for c in chunks for p in fwd(c)[2]]
    assert torch.equal(_u8(outs), _u8(want))
