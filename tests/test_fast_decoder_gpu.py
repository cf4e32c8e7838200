"""GPU tests of the decoder's fast mode (one fp16 operand plane, ops.H1: one wgmma per product).

Op level, every one-plane path of the convolution (row reuse, per-tap, KC = 32, split-K with the finalize kernel and with the
fused post kernel, post-op through emo_apply, sub-pixel up-convolution, residual with res_shift, GroupNorm statistics):
  * within accumulation error (1e-5 of the scale) of float64 evaluated on the ROUNDED operands, fp16(x * 16) / 16 and
    fp16(w * 256) / 256: the kernel adds nothing but its chunked fp32 accumulation to the format's own error;
  * within the one-plane operand bound of float64 on the fp32 operands: each product is off by at most (2^-11 + 2^-11 +
    2^-22) of |x| |w|, so |error| <= 2^-10 conv(|x|, |w|) (+ the accumulation term);
  * the post-op's one fp16 plane is fp16(16 y) of the float64 post-op output to within its rounding;
  * the accumulation bias of the one-plane chunks (16 MMAs) stays ~1e-6 relative, a single chain is the negative control.
The one fp16 planes written by ops.apply, ops.grid_sample3d and ops.split_bf16 are bit-equal to fp16(y * 16) of their fp32
output.  Decoder in isolation, fed the oracle's aligned_volume (as tests/test_stage_parity_gpu.py::test_decoder): image
max-abs <= 3.5e-3, mean-abs <= 4e-4, logits max-abs <= 1.6e-2 at 256^2 and 512^2 (bounds from tools/decoder_precision_emulation.py:
2.0e-3 / 3.3e-3, 2.2e-4 / 2.9e-4, 8.5e-3 / 1.5e-2).  End to end, InferenceWrapper(precision="fast") against "exact": every
uint8 pixel within one level (max-abs < 1/255), PSNR >= 60 dB, two runs bit-identical and four frames in flight equal to eager."""
import math

import pytest
import torch
import torch.nn.functional as F

import conv_plan_cases as CP
from oracle import frames as FR

pytestmark = pytest.mark.gpu
H1 = "h1"
ACC_TOL = 1e-5       # vs float64 on the rounded operands, relative to max(1, scale)


@pytest.fixture(scope="module")
def ops():
    from emoportraits_b200 import ops as o
    return o


def _round(x, scale):
    return (x.float() * scale).half().double() / scale


def _upconv_ref(x, wf):
    """float64 sub-pixel up-convolution: x (N, Ci, H, W) low resolution, wf (4 phases, 2, 2, Co, Ci) folded weights"""
    N, _, H, W = x.shape
    xp = F.pad(x, (1, 1, 1, 1))
    out = torch.zeros((N, wf.shape[3], 2 * H, 2 * W), dtype=torch.float64, device=x.device)
    for a in (0, 1):
        for b in (0, 1):
            k = wf[2 * a + b].permute(2, 3, 0, 1)   # (Co, Ci, 2, 2)
            out[:, :, a::2, b::2] = F.conv2d(xp, k)[:, :, a:a + H, b:b + W]
    return out


def _reference(c, x, w, b, res, ops):
    """(float64 result on the rounded operands, on the fp32 operands, the operand bound 2^-10 conv(|x|, |w|), scale)"""
    xr = _round(x, ops.F16_ACT_SCALE)
    if c.upconv:
        wf = ops.fold_upconv_weight(w.cpu()).to(x.device)
        wfr = _round(wf, ops.F16_W_SCALE)
        y_r, y_x = _upconv_ref(xr, wfr), _upconv_ref(x.double(), wf.double())
        absb = _upconv_ref(x.double().abs(), wf.double().abs())
    else:
        nd = len(c.sp)
        conv = F.conv3d if nd == 3 else F.conv2d
        wr = _round(w, ops.F16_W_SCALE)
        kw = dict(stride=c.stride, padding=c.k // 2)
        y_r, y_x, absb = conv(xr, wr, **kw), conv(x.double(), w.double(), **kw), conv(x.double().abs(), w.double().abs(), **kw)
    extra = 0
    if b is not None:
        extra = extra + b.double().view((1, -1) + (1,) * (y_r.dim() - 2))
    if res is not None:
        r = res.double()
        if c.res_shift:
            r = F.interpolate(r, scale_factor=2, mode="nearest")
        extra = extra + r
    y_r, y_x = y_r + extra, y_x + extra
    scale = max(y_r.abs().max().item(), 1.0)
    return y_r, y_x, absb * 2.0 ** -10, scale


def _args(c, ops, x, w, b, res, stats=None, post=None):
    pw = (ops.pack_upconv_weight(w.cpu(), device="cuda", planes=H1) if c.upconv
          else ops.pack_conv_weight(w.cpu(), device="cuda", planes=H1))
    a = ops.split_bf16(CP.cl(x), H1)
    s3 = (c.stride,) * 3 if len(c.sp) == 3 else (1, c.stride, c.stride)
    kw = dict(stride=s3, bias=b, residual=CP.cl(res) if res is not None else None, res_shift=c.res_shift, stats=stats, G=c.G,
              split_k=c.split_k, upconv=c.upconv, post=post)
    return a, pw, kw


def _to_ref_layout(c, t):
    t = t.permute(0, 4, 1, 2, 3)
    return t if len(c.sp) == 3 else t[:, :, 0]


# plan class at 132 SMs -> case: every one-plane kernel, both main loops, all three split-K finishes, statistics, residual
# (one-plane halo tiles are half the size: row reuse always finds room for an A ring of three)
CASES = [
    ("h1<64,1> BN128 rr3 none", CP.Case("", 64, 128, (96, 96), planes=H1, residual=True, stats=True)),
    ("h1<64,1> BN128 rr3 apply", CP.Case("", 128, 256, (64, 80), planes=H1, post=True, stats=True)),
    ("h1<64,1> BN128 tap none", CP.Case("", 512, 128, (96, 96), k=1, planes=H1, stats=True)),
    ("h1<64,1> BN128 tap finalize", CP.Case("", 256, 256, (8, 8), planes=H1, residual=True, stats=True)),
    ("h1<64,1> BN128 tap finalize+apply", CP.Case("", 128, 128, (32, 32), planes=H1, post=True, stats=True)),
    ("h1<64,1> BN128 tap post", CP.Case("", 256, 256, (8, 8), planes=H1, post=True, stats=True)),
    ("h1<32,1> BN96 rr3 none", CP.Case("", 96, 96, (96, 96), planes=H1, residual=True, res_shift=1, stats=True)),
    ("h1<32,1> BN96 tap none", CP.Case("", 160, 96, (96, 96), k=1, planes=H1)),
    ("h1ps<64,1> BN128 rr3 none", CP.Case("", 128, 128, (64, 64), planes=H1, upconv=True, stats=True)),
    ("h1ps<64,1> BN64 rr3 none", CP.Case("", 256, 64, (48, 40), planes=H1, upconv=True, residual=True, res_shift=1, stats=True)),
    # the 160 / 320 and 96 / 192 channel layers of the 256^2 / 512^2 decoders
    ("h1<64,1> BN80 rr3 none", CP.Case("", 64, 160, (96, 40), planes=H1, residual=True, stats=True)),
    ("h1<64,1> BN80 rr3 apply", CP.Case("", 64, 160, (96, 40), planes=H1, post=True, stats=True)),
    ("h1<64,1> BN80 tap none", CP.Case("", 64, 160, (96, 40), k=1, planes=H1)),
    ("h1<64,1> BN96 rr3 none", CP.Case("", 64, 192, (96, 40), planes=H1, residual=True)),
    ("h1<64,1> BN96 rr3 apply", CP.Case("", 64, 192, (96, 40), planes=H1, post=True, stats=True)),
    ("h1<64,1> BN96 tap none", CP.Case("", 64, 192, (96, 40), k=1, planes=H1, stats=True)),
    ("h1<32,1> BN80 rr3 none", CP.Case("", 160, 160, (96, 40), planes=H1, residual=True, stats=True)),
    ("h1<32,1> BN80 rr3 apply", CP.Case("", 32, 160, (96, 40), planes=H1, post=True, stats=True)),
    ("h1<32,1> BN96 rr3 apply", CP.Case("", 160, 96, (96, 96), planes=H1, post=True, stats=True)),
    ("h1ps<64,1> BN80 rr3 none", CP.Case("", 64, 160, (24, 40), planes=H1, upconv=True, residual=True, stats=True)),
    ("h1ps<64,1> BN96 rr3 none", CP.Case("", 64, 96, (48, 48), planes=H1, upconv=True, residual=True, res_shift=1)),
]


def _plan_class(info):
    from emoportraits_b200 import lib as L

    loop = f"rr{info.sa}" if info.yreuse else "tap"
    return f"{L.conv_kernel_name(info.kernel)} BN{info.BN} {loop} {L.CONV_FINISH[info.finish]}"


@pytest.mark.parametrize("want,c", CASES, ids=[w for w, _ in CASES])
def test_one_plane_conv_against_float64(ops, want, c):
    torch.manual_seed(0)
    x, w, b, res, _ = CP.make(c, "cuda")
    st = torch.zeros((c.N, c.G, 2), dtype=torch.float64, device="cuda") if c.stats else None
    Do, Ho, Wo = CP.out_shape(c)
    post = None
    if c.post:
        gamma = torch.linspace(0.5, 1.5, c.Cout, device="cuda")
        beta = torch.linspace(-0.5, 0.5, c.Cout, device="cuda")
        post = dict(act=ops.ACT_RELU, planes=H1, want_f32=True, want_split=True,
                    gn=dict(stats=st, count=Do * Ho * Wo * c.Cout / c.G, gamma=gamma, beta=beta))
    a, pw, kw = _args(c, ops, x, w, b, res, st, post)
    info = ops.conv_plan(a, pw, **kw)
    assert info.NP == 1 and info.fp16 == 1
    if torch.cuda.get_device_properties(0).multi_processor_count == CP.SM_COUNT:
        assert _plan_class(info) == want, (_plan_class(info), want)
    got = ops.conv_igemm(a, pw, **kw)
    torch.cuda.synchronize()
    y_r, y_x, opb, scale = _reference(c, x, w, b, res, ops)
    msg = f"\n[{want}] ksplit {info.ksplit}:"
    if c.post:
        pout, psp = got
        pref = CP.post_reference(c, y_r, c.G)
        pe = (_to_ref_layout(c, pout).double() - pref).abs().max().item()
        # the post-op's one fp16 plane: fp16(16 y) of the float64 post-op output, up to fp16 rounding and the post-op's own error
        plane = _to_ref_layout(c, psp.hi.float()).double() / ops.F16_ACT_SCALE
        ple = ((plane - pref).abs() - 2.0 ** -11 * pref.abs()).max().item()
        msg += f" post-op max-abs {pe:.2e}, one-plane post-op excess over fp16 rounding {ple:.2e}"
        assert pe < 5e-5 * max(1.0, pref.abs().max().item()), pe
        assert ple < 5e-5 * max(1.0, pref.abs().max().item()), ple
    else:
        out = _to_ref_layout(c, got).double()
        e_acc = (out - y_r).abs().max().item()
        excess = ((out - y_x).abs() - opb).max().item()
        msg += (f" vs rounded operands {e_acc:.2e} ({e_acc / scale:.1e} of scale {scale:.1f}); vs fp32 operands "
                f"{(out - y_x).abs().max().item():.2e}, excess over the operand bound {excess:.1e}")
        assert e_acc < ACC_TOL * scale, (e_acc, scale)
        assert excess < ACC_TOL * scale, excess
    if st is not None:
        r = y_r.reshape(c.N, c.G, -1)
        count = r.shape[-1]
        d_mean = (st[..., 0] / count - r.mean(-1)).abs().max().item()
        msq = (r * r).mean(-1)
        d_msq = ((st[..., 1] / count - msq).abs() / msq).max().item()
        msg += f" stats: mean {d_mean:.1e} mean-square {d_msq:.1e} (rel)"
        assert d_mean < 1e-6 * scale and d_msq < 1e-5, (d_mean, d_msq)
    print(msg)


# accumulation bias of the one-plane chunks (16 MMAs = 256 channels of K per chunk, emo_conv_plan's default for NP = 1).
# H100 SXM: 16-MMA chunks -1.1e-6 / -1.2e-6 (1x1 x 1536 / 3x3 x 512; 400 W card), 32-MMA chunks -2.6e-6 / -2.7e-6 (700 W card),
# one chain -9.2e-6 / -2.9e-5
BIAS_BOUND = 2e-6
CONTROL_FACTOR = 3.0


@pytest.mark.parametrize("Cin,k", [(1536, 1), (512, 3)])
def test_one_plane_accumulation_bias(ops, Cin, k):
    c = CP.Case("", Cin, 128, (32, 32), k=k, planes=H1, split_k=False, bias=False)
    x, w, _, _, _ = CP.make(c, "cuda", positive=True)
    y_r, _, _, _ = _reference(c, x, w, None, None, ops)

    def bias(acc):
        a, pw, kw = _args(c, ops, x, w, None, None)
        out = ops.conv_igemm(a, pw, acc_chunk_mmas=acc, **kw)
        torch.cuda.synchronize()
        return ((_to_ref_layout(c, out).double() - y_r).mean() / y_r.abs().mean()).item()

    b_def, b_one = bias(0), bias(1 << 20)
    print(f"\n[one-plane accumulation bias {Cin} ch k{k}] default chunks {b_def:+.2e}, one chain {b_one:+.2e} (relative to mean |ref|)")
    assert abs(b_def) < BIAS_BOUND, b_def
    assert b_one < -BIAS_BOUND and abs(b_one) > CONTROL_FACTOR * abs(b_def), (b_def, b_one)


# ------------------------------------------------------------------------------------------------------------------
def _bits_equal(plane, y, scale):
    want = (y * scale).half()
    return torch.equal(plane.view(torch.int16), want.view(torch.int16))


@pytest.mark.parametrize("C,up", [(64, 1), (64, 2), (12, 1), (12, 2)])   # C % 8 == 0: two float4 per thread, else one
def test_apply_one_plane_bits(ops, C, up):
    torch.manual_seed(1)
    x = torch.randn(2, 1, 24, 20, C, device="cuda") * 3
    A = torch.rand(2, C, device="cuda") + 0.5
    B = torch.randn(2, C, device="cuda")
    out, sp = ops.apply(x, A, B, act=ops.ACT_RELU, up=up, want_f32=True, want_split=True, planes=H1)
    assert sp.lo is None and sp.hi.dtype == torch.float16
    assert _bits_equal(sp.hi, out, ops.F16_ACT_SCALE)
    _, sp2 = ops.apply(x, A, B, act=ops.ACT_NONE, up=up, want_f32=True, want_split=True, planes=ops.H2)   # two planes unchanged
    assert sp2.lo is not None


def test_split_one_plane_bits(ops):
    x = torch.randn(3, 1, 16, 16, 96, device="cuda") * 4
    sp = ops.split_bf16(x, H1)
    assert sp.lo is None and _bits_equal(sp.hi, x, ops.F16_ACT_SCALE)


@pytest.mark.parametrize("in_layout,out_layout", [("cl", "hwdc"), ("cl", "cl"), ("cl", "ncdhw"), ("ncdhw", "hwdc")])
def test_grid_sample3d_one_plane_bits(ops, in_layout, out_layout):
    torch.manual_seed(2)
    N, Cc, D, H, W = 1, 32, 8, 24, 24
    vol = torch.randn(N, D, H, W, Cc, device="cuda") if in_layout == "cl" else torch.randn(N, Cc, D, H, W, device="cuda")
    theta = torch.tensor([[[0.9, 0.1, 0.0, 0.05], [-0.1, 0.9, 0.0, 0.0], [0.0, 0.0, 1.0, 0.02]]], device="cuda")
    out, sp = ops.grid_sample3d(vol, theta=theta, out_size=(D, H, W), in_layout=in_layout, out_layout=out_layout,
                                want_f32=True, want_split=True, planes=H1)
    assert sp.lo is None and _bits_equal(sp.hi, out, ops.F16_ACT_SCALE)


# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=[256, 512])
def dec_ctx(request):
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import Model
    from oracle import restatement as R

    size = request.param
    cfg = shipped_config(size)
    sd, hsd = synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0)
    ocfg = R.config_from_state_dict(sd, size)
    with torch.no_grad():
        taps = {}
        R.driver_pass(sd, hsd, R.source_pass(sd, hsd, FR.frame(size, 21, "noise"), ocfg), FR.frame(size, 22, "noise"), ocfg, taps)
    return dict(size=size, cfg=cfg, sd=sd, hsd=hsd, taps=taps, model=Model(cfg, sd, hsd, "cuda", precision="fast"))


def test_fast_decoder_against_oracle(ops, dec_ctx):
    cfg, taps = dec_ctx["cfg"], dec_ctx["taps"]
    av = taps["aligned_volume"]
    hwdc = av[0].permute(2, 3, 1, 0).contiguous().view(1, 1, cfg.S, cfg.S, cfg.D * cfg.C).cuda()
    dec = dec_ctx["model"].decoder_nw
    assert dec.planes == H1
    logits, _, _ = dec(ops.split_bf16(hwdc, H1), want_logits=True)
    img, _, _ = dec(ops.split_bf16(hwdc, H1))
    ref_logits = taps["logits"]
    ref_img = torch.sigmoid(ref_logits)
    e_img = (img.cpu() - ref_img).abs()
    e_log = (logits.cpu() - ref_logits).abs().max().item()
    print(f"\n[fast decoder @{dec_ctx['size']}] image max-abs {e_img.max().item():.2e} mean-abs {e_img.mean().item():.2e}, "
          f"logits max-abs {e_log:.2e}")
    assert e_img.max().item() <= 3.5e-3 and e_img.mean().item() <= 4e-4 and e_log <= 1.6e-2


def test_fast_wrapper_end_to_end(dec_ctx, tmp_path):
    """InferenceWrapper(precision="fast") against "exact" on the fixture frames; two runs and four frames in flight"""
    import pathlib

    from emoportraits_b200.infer import InferenceWrapper

    size, cfg = dec_ctx["size"], dec_ctx["cfg"]
    gold = pathlib.Path(__file__).parent / "golden"
    exp = tmp_path / "logs" / "exp" / "checkpoints"
    exp.mkdir(parents=True)
    (tmp_path / "logs" / "exp" / "args.txt").write_text((gold / f"args_{size}.txt").read_text())
    torch.save(dec_ctx["sd"], exp / "000_model.pth")
    kw = dict(experiment_name="exp", model_file_name="000_model.pth", project_dir=str(tmp_path), folder="logs",
              print_params=False, head_pose_state_dict=dec_ctx["hsd"])
    exact, fast = InferenceWrapper(**kw), InferenceWrapper(precision="fast", **kw)
    src = FR.pil(size, 21, "smooth")
    drv = [FR.pil(size, 60 + i, "smooth") for i in range(5)]
    fw = dict(crop=False, mix=True, mix_old=False)
    _, img_e = exact.forward(src, drv, **fw)
    pil_f, img_f = fast.forward(src, drv, **fw)
    _, img_f2 = fast.forward(None, drv, **fw)
    err = (img_f - img_e).abs()
    psnr = [10 * math.log10(1.0 / ((img_f[i] - img_e[i]) ** 2).mean().item()) for i in range(len(drv))]
    print(f"\n[fast vs exact @{size}] image max-abs {err.max().item():.2e} mean-abs {err.mean().item():.2e}, "
          f"PSNR min {min(psnr):.1f} dB")
    assert err.max().item() < 1.0 / 255
    assert min(psnr) >= 60.0
    assert torch.equal(img_f, img_f2)            # two runs bit-identical
    # four frames in flight (the list form) equal the eager driver pass
    model = fast.model
    eager = torch.cat([model.driver_pass(fast._state, fast._prep(d), mix=True, mix_old=False)[0] for d in drv])
    e_fl = [(img_f[i] - eager[i]).abs().max().item() for i in range(len(drv))]
    print(f"[fast @{size}] four in flight vs eager {e_fl}")
    assert max(e_fl) < 5e-4 and sum(e == 0.0 for e in e_fl) >= len(e_fl) - 1, e_fl
