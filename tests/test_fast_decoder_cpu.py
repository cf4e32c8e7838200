"""CPU tests of the decoder's fast mode (one fp16 operand plane, ops.H1):
  * in EMO_DRY_RUN mode the stage-1 driver pass with precision="fast" plans every decoder convolution on a one-plane kernel
    (NP = 1), the sub-pixel up-convolutions and (at 256^2) the split-K layers with a post-op included, at 256^2 and 512^2, and
    feeds the decoder one fp16 plane from grid_sample3d; every other network keeps its two-plane operands;
  * every one-plane case of tests/test_fast_decoder_gpu.py reaches the plan class it names at 132 SMs;
  * emo_conv_plan / emo_apply / emo_grid_sample3d refuse the invalid one-plane combinations;
  * the header's kernel ids match the binding;
  * `precision=` of Model and InferenceWrapper."""
import ctypes as C
import pathlib
import subprocess

import pytest
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
H1_KERNELS = {"h1<64,1>", "h1<32,1>", "h1ps<64,1>"}


@pytest.fixture
def dry(monkeypatch):
    from emoportraits_b200 import lib as L

    monkeypatch.setattr(L, "DRY_RUN", True)   # host tensors are accepted as operands; nothing is launched
    return L


def _record_driver_pass(L, monkeypatch, size, precision):
    """(plans of the decoder's convolutions, plans of every other convolution, grid_sample3d descriptors) of one dry-run
    driver pass; a plan is (emo_conv_plan return code, ConvPlanInfo, upconv, post)"""
    from emoportraits_b200 import nets
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import Model

    lib = L.load()
    rec = dict(dec=[], other=[], gs=[])
    in_dec = [False]
    launch = L.call

    def call(name, *args):
        if name == "emo_conv_igemm":
            d = args[0]._obj
            info = L.ConvPlanInfo()
            rc = lib.emo_conv_plan(C.byref(d), 132, C.byref(info))
            rec["dec" if in_dec[0] else "other"].append((rc, info, bool(d.upconv), bool(d.post), d.operand_fp16, d.a_lo))
        elif name == "emo_grid_sample3d":
            d = args[0]._obj
            rec["gs"].append((d.plane_fp16, d.plane_scale, d.out_hi, d.out_lo, d.os_c))
        return launch(name, *args)

    dec_call = nets.Decoder.__call__

    def decoder(self, *a, **k):
        in_dec[0] = True
        try:
            return dec_call(self, *a, **k)
        finally:
            in_dec[0] = False

    monkeypatch.setattr(L, "call", call)
    monkeypatch.setattr(nets.Decoder, "__call__", decoder)
    cfg = shipped_config(size)
    model = Model(cfg, synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0), "cpu", precision=precision)
    x = torch.rand(1, 3, size, size)
    st = model.source_pass(x)
    for k in rec:
        rec[k].clear()
    model.driver_pass(st, x, mix=True)
    return model, rec


@pytest.mark.parametrize("size,split_post", [(256, True), (512, False)])   # the 512^2 decoder has no split-K layer
def test_fast_mode_plans_every_decoder_conv_on_one_plane(dry, monkeypatch, size, split_post):
    from emoportraits_b200 import ops

    model, rec = _record_driver_pass(dry, monkeypatch, size, "fast")
    assert model.decoder_nw.planes == ops.H1 and model.precision["warp"] == ops.H2
    dec = rec["dec"]
    assert dec, "no decoder convolution recorded"
    refused = [i for i, r in enumerate(dec) if r[0] != 0]
    assert not refused, refused
    kinds = [dry.conv_kernel_name(info.kernel) for _, info, *_ in dec]
    print(f"\n[fast decoder @{size}] {len(dec)} convolutions: " + ", ".join(f"{k} x{kinds.count(k)}" for k in sorted(set(kinds))))
    assert all(info.NP == 1 and info.fp16 == 1 for _, info, *_ in dec)
    assert set(kinds) <= H1_KERNELS, set(kinds)
    ups = [r for r in dec if r[2]]
    assert ups and all(dry.conv_kernel_name(r[1].kernel) == "h1ps<64,1>" for r in ups)
    finishes = {dry.CONV_FINISH[r[1].finish] for r in dec}
    print(f"[fast decoder @{size}] finishes {sorted(finishes)}")
    assert bool(finishes & {"post", "finalize+apply"}) == split_post, finishes   # split-K with a post-op
    # the decoder's input: ONE fp16 plane of the aligned volume (x16) in the (h, w, d, c) layout
    plane_fp16, scale, hi, lo, os_c = rec["gs"][-1]
    assert plane_fp16 == 1 and scale == ops.F16_ACT_SCALE and hi and not lo and os_c == 1
    # every other network keeps its operands (two fp16 planes, H2)
    other = rec["other"]
    assert other and all(r[0] == 0 and r[1].NP == 2 for r in other)


@pytest.mark.parametrize("size", [256])
def test_exact_mode_plans_unchanged(dry, monkeypatch, size):
    model, rec = _record_driver_pass(dry, monkeypatch, size, "exact")
    assert model.decoder_nw.planes == 2
    assert rec["dec"] and all(r[0] == 0 and r[1].NP == 2 and r[1].fp16 == 0 for r in rec["dec"])
    assert rec["gs"][-1][0] == 0 and rec["gs"][-1][3]


# ------------------------------------------------------------------------------------------------------------------
def _one_plane_desc(ops, upconv=False, Cin=64, Cout=64):
    """a valid one-plane descriptor (host tensors), with the objects it points to"""
    x = ops.Split.empty((1, 1, 16, 16, Cin), "cpu", ops.H1)
    w = torch.randn(Cout, Cin, 3, 3) * 0.05
    pw = ops.pack_upconv_weight(w, device="cpu", planes=ops.H1) if upconv else ops.pack_conv_weight(w, device="cpu", planes=ops.H1)
    d, ret, pd, _ = ops._conv_desc(x, pw, (1, 1, 1), None, None, None, 0, 0, None, False, None, 32, None, 0, False, upconv, None)
    return d, (x, pw, ret, pd)


def _plan(L, d):
    info = L.ConvPlanInfo()
    return L.load().emo_conv_plan(C.byref(d), 132, C.byref(info)), info


@pytest.mark.parametrize("upconv", [False, True])
def test_one_plane_plan_reports_np1(dry, upconv):
    from emoportraits_b200 import ops

    d, keep = _one_plane_desc(ops, upconv)
    rc, info = _plan(dry, d)
    assert rc == 0 and info.NP == 1 and info.fp16 == 1
    assert dry.conv_kernel_name(info.kernel) == ("h1ps<64,1>" if upconv else "h1<64,1>")
    assert info.flush * (info.KC // 16) == 16          # the one-plane default accumulation chunk: 16 MMAs


def test_one_plane_invalid_combinations_are_refused(dry):
    from emoportraits_b200 import ops

    d, keep = _one_plane_desc(ops)
    buf = torch.zeros(1 << 16, dtype=torch.float16)   # a 16-byte aligned stand-in plane (never read: refused first)
    cases = {
        "a_lo2 with one plane": dict(a_lo2=buf.data_ptr(), w_lo2=buf.data_ptr()),
        "one plane without operand_fp16": dict(operand_fp16=0),
        "a one plane, w two": dict(w_lo=buf.data_ptr()),
        "a two planes, w one": dict(a_lo=buf.data_ptr()),
    }
    for name, fields in cases.items():
        dd = type(d).from_buffer_copy(d)
        for k, v in fields.items():
            setattr(dd, k, v)
        rc, _ = _plan(dry, dd)
        assert rc == -1, (name, rc)
    # two fp16 planes still take no upconv
    x = ops.Split.empty((1, 1, 16, 16, 64), "cpu", ops.H2)
    du, keep2 = _one_plane_desc(ops, upconv=True)
    du.a_lo, du.w_lo = x.lo.data_ptr(), x.lo.data_ptr()
    assert _plan(dry, du)[0] == -1


def test_one_plane_apply_and_grid_sample_refuse_bad_planes(dry):
    """argument checks run before any CUDA call: emo_apply / emo_grid_sample3d with one fp16 plane"""
    lib = dry.load()
    buf = torch.zeros(1 << 12, dtype=torch.float32)
    p = buf.data_ptr()
    # emo_apply: out_hi alone needs plane_fp16; plane_fp16 takes no out_lo2 and needs a positive scale
    for hi, lo, lo2, f16, scale in [(p, None, None, 0, 0.0), (p, p, p, 1, 16.0), (p, None, None, 1, 0.0), (None, p, None, 1, 16.0)]:
        d = dry.ApplyDesc(x=p, N=1, C=8, D=1, H=4, W=4, act=0, up=1, out_hi=hi, out_lo=lo, out_lo2=lo2, plane_fp16=f16,
                          plane_scale=scale)
        assert lib.emo_apply(C.byref(d), None) == -1, (hi, lo, lo2, f16, scale)
    # emo_grid_sample3d: plane_fp16 writes out_hi alone (no out_lo / out_lo2) and needs a positive scale
    for lo, lo2, scale in [(p, None, 16.0), (None, p, 16.0), (None, None, 0.0)]:
        d = dry.GridSample3dDesc(in_=p, in_layout=1, N=1, C=8, Din=2, Hin=2, Win=2, theta=p, Dout=2, Hout=2, Wout=2,
                                 out_hi=p, out_lo=lo, out_lo2=lo2, os_n=64, os_c=1, os_d=8, os_h=16, os_w=8, plane_fp16=1,
                                 plane_scale=scale)
        assert lib.emo_grid_sample3d(C.byref(d), None) == -1, (lo, lo2, scale)


def test_header_kernel_ids_match_the_binding(tmp_path):
    """every EMO_CONV_KERNEL_* id (the one-plane ids follow implicitly) names the binding's kernel of that id"""
    import re

    from emoportraits_b200 import lib as L

    hdr = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "emoportraits_b200.h").read_text(), flags=re.S)
    start = hdr.index("EMO_CONV_KERNEL_BF16X2_KC64")
    names = re.findall(r"\bEMO_CONV_KERNEL_\w+", hdr[start:hdr.index("};", start)])
    src = tmp_path / "ids.c"
    src.write_text(f'#include <stdio.h>\n#include "{ROOT / "include" / "emoportraits_b200.h"}"\nint main(void) {{\n'
                   + "".join(f'  printf("{n} %d\\n", (int){n});\n' for n in names) + "  return 0;\n}\n")
    exe = tmp_path / "ids"
    subprocess.run(["gcc", "-std=c11", "-o", str(exe), str(src)], check=True)
    ids = dict(ln.split() for ln in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    ids = {n: int(v) for n, v in ids.items()}
    assert sorted(ids.values()) == list(range(len(L.CONV_KERNELS) + len(L.CONV_KERNELS_H1)))
    assert ids["EMO_CONV_KERNEL_H1_KC64"] == 7 and ids["EMO_CONV_KERNEL_H1_KC32"] == 8 and ids["EMO_CONV_KERNEL_H1_UPCONV_KC64"] == 9
    for n, v in ids.items():
        name = L.conv_kernel_name(v)
        if v >= len(L.CONV_KERNELS):
            want = {"h1<64,1>": "H1_KC64", "h1<32,1>": "H1_KC32", "h1ps<64,1>": "H1_UPCONV_KC64"}[name]
            assert n == "EMO_CONV_KERNEL_" + want, (n, v, name)


# ------------------------------------------------------------------------------------------------------------------
def test_model_precision_presets():
    from emoportraits_b200 import ops
    from emoportraits_b200.infer import Model

    assert Model.resolve_precision(None) == Model.PRECISION == Model.resolve_precision("exact")
    fast = Model.resolve_precision("fast")
    assert fast == dict(Model.PRECISION, decoder=ops.H1)
    assert Model.resolve_precision(dict(decoder=ops.H1)) == fast
    assert Model.resolve_precision(dict(decoder=3))["decoder"] == 3
    for bad in ("turbo", "FAST", dict(decoder=ops.H2), dict(warp=ops.H1), dict(expression=ops.H1, decoder=ops.H1)):
        with pytest.raises(ValueError):
            Model.resolve_precision(bad)


def test_inference_wrapper_precision_argument():
    from emoportraits_b200.infer import InferenceWrapper

    with pytest.raises(ValueError, match="precision"):
        InferenceWrapper("x", precision="turbo")
    with pytest.raises(ValueError, match="precision"):
        InferenceWrapper("x", precision=None)
    if not torch.cuda.is_available():   # a valid setting passes the check and reaches the device requirement
        with pytest.raises(RuntimeError, match="CUDA"):
            InferenceWrapper("x", precision="fast")


def test_one_plane_host_formats():
    from emoportraits_b200 import ops

    w = torch.randn(32, 64, 3, 3) * 0.05
    pw = ops.pack_conv_weight(w, device="cpu", planes=ops.H1)
    assert pw.f16 and pw.lo is None and pw.lo2 is None and pw.hi.dtype == torch.float16 and pw.scale == ops.F16_W_SCALE
    ref = torch.zeros(9, 32, 64)
    ref[:, :32] = w.permute(2, 3, 0, 1).reshape(9, 32, 64)
    assert torch.equal(pw.hi, (ref * ops.F16_W_SCALE).half())
    pu = ops.pack_upconv_weight(w, device="cpu", planes=ops.H1)
    assert pu.lo is None and torch.equal(pu.hi, (ops.fold_upconv_weight(w).reshape(16, 32, 64) * ops.F16_W_SCALE).half())
    sp = ops.Split.empty((1, 1, 4, 4, 8), "cpu", ops.H1)
    assert sp.planes == 1 and sp.f16 and sp.lo is None and sp.scale == ops.F16_ACT_SCALE and sp.hi.dtype == torch.float16
    v = sp.view(1, 1, 16, 8)
    assert v.lo is None and v.shape == (1, 1, 16, 8)
    sp.hi.fill_(3.0)
    assert torch.equal(sp.float(), torch.full((1, 1, 4, 4, 8), 3.0 / ops.F16_ACT_SCALE))


def test_gpu_cases_reach_their_plan_class(dry):
    """the one-plane cases of tests/test_fast_decoder_gpu.py plan as they say at 132 SMs (H100 SXM)"""
    import conv_plan_cases as CP
    import test_fast_decoder_gpu as T
    from emoportraits_b200 import ops

    bad = []
    for want, c in T.CASES:
        x, w, b, res, _ = CP.make(c, "cpu")
        st = torch.zeros((c.N, c.G, 2), dtype=torch.float64) if c.stats else None
        post = None
        if c.post:
            post = dict(act=ops.ACT_RELU, planes=ops.H1, want_f32=True, want_split=True,
                        gn=dict(stats=st, count=1.0, gamma=torch.ones(c.Cout), beta=torch.zeros(c.Cout)))
        pw = (ops.pack_upconv_weight(w, device="cpu", planes=ops.H1) if c.upconv
              else ops.pack_conv_weight(w, device="cpu", planes=ops.H1))
        a = ops.Split.empty(CP.cl(x).shape, "cpu", ops.H1)
        info = ops.conv_plan(a, pw, stride=(1, c.stride, c.stride), bias=b, residual=CP.cl(res) if res is not None else None,
                             res_shift=c.res_shift, stats=st, G=c.G, split_k=c.split_k, upconv=c.upconv, post=post,
                             sm_count=CP.SM_COUNT)
        if T._plan_class(info) != want:
            bad.append((want, T._plan_class(info)))
    assert not bad, bad
