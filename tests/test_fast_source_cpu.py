"""CPU tests of the source pass's fast mode (InferenceWrapper(source_precision="fast"), Model.SOURCE_FAST):
  * in EMO_DRY_RUN mode, at 256^2 and 512^2, every LocalEncoder / VolumeSource / Unet3D convolution plans on a one-plane
    kernel (EMO_CONV_KERNEL_H1_*), none is refused, and each falls in a plan class that tests/test_fast_source_gpu.py (3-D
    layers; 2-D layers also tests/test_fast_decoder_gpu.py / tests/test_fast_stage2_gpu.py) sweeps on the GPU;
  * the local encoder's stem is emo_stem_pack + one emo_conv_igemm writing GroupNorm statistics, and no emo_conv_direct;
  * the identity / expression / head-pose / xy-warp launches of the source pass and the whole driver pass issue the same
    descriptors as in exact mode;
  * every case of tests/test_fast_source_gpu.py reaches the plan class it names at 132 SMs;
  * `source_precision=` of InferenceWrapper and the one-plane overrides Model.resolve_precision accepts and refuses."""
import ctypes as C

import pytest
import torch

import conv_plan_cases as CP

SOURCE_NETS = ("LocalEncoder", "VolumeSource", "Unet3D")


@pytest.fixture
def dry(monkeypatch):
    from emoportraits_b200 import lib as L

    monkeypatch.setattr(L, "DRY_RUN", True)   # host tensors are accepted as operands; nothing is launched
    return L


def _fields(d):
    """the scalar fields and the NULL-ness of the pointer fields of a ctypes descriptor"""
    out = []
    for name, typ in d._fields_:
        v = getattr(d, name)
        out.append((name, v is not None and v != 0) if typ is C.c_void_p else (name, v))
    return tuple(out)


def _record(L, monkeypatch, size, precision):
    """(model, source-pass calls, driver-pass calls) of one dry-run Model; a call is (network, C-ABI name, descriptor
    fields or None, conv plan or None), network the source network class that issued it or "" for the rest; a plan is
    (emo_conv_plan return code, ConvPlanInfo, emo_conv_desc copy) at 132 SMs"""
    from emoportraits_b200 import nets
    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.infer import Model

    lib = L.load()
    calls = []
    where = [""]
    launch = L.call

    def call(name, *args):
        plan = None
        if args and hasattr(args[0], "_obj"):          # a descriptor passed by reference
            d = args[0]._obj
            fields = _fields(d)
            if name == "emo_conv_igemm":
                info = L.ConvPlanInfo()
                plan = (lib.emo_conv_plan(C.byref(d), 132, C.byref(info)), info, type(d).from_buffer_copy(d))
                if d.post:
                    fields += _fields(C.cast(d.post, C.POINTER(L.ApplyDesc)).contents)
        else:                                          # scalar arguments: device pointers are data_ptr() values
            fields = tuple(a.value if isinstance(a, C.c_float) else "ptr" if isinstance(a, int) and a > 1 << 20 else a
                           for a in args)
        calls.append((where[0], name, fields, plan))
        return launch(name, *args)

    for cls in SOURCE_NETS:
        orig = getattr(nets, cls).__call__

        def scoped(self, *a, _orig=orig, _cls=cls, **k):
            where[0] = _cls
            try:
                return _orig(self, *a, **k)
            finally:
                where[0] = ""
        monkeypatch.setattr(getattr(nets, cls), "__call__", scoped)
    monkeypatch.setattr(L, "call", call)
    cfg = shipped_config(size)
    model = Model(cfg, synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0), "cpu", precision=precision)
    torch.manual_seed(0)
    x = torch.rand(1, 3, size, size)
    st = model.source_pass(x)
    src_calls = list(calls)
    calls.clear()
    model.driver_pass(st, x, mix=True)
    return model, src_calls, list(calls)


def _source_fast():
    from emoportraits_b200.infer import Model

    return dict(Model.SOURCE_FAST)


def _swept_classes():
    import test_fast_decoder_gpu as TD
    import test_fast_source_gpu as TF
    import test_fast_stage2_gpu as TS

    two_d = {w for w, _ in TD.CASES} | {w for w, _ in TS.CASES}
    return two_d | {w for w, _ in TF.CASES} | {TF.DEPTH_CASE[0]}


@pytest.mark.parametrize("size", [256, 512])
def test_fast_source_plans_every_source_conv_on_one_plane(dry, monkeypatch, size):
    import test_fast_source_gpu as TF
    from emoportraits_b200 import ops

    model, calls, _ = _record(dry, monkeypatch, size, _source_fast())
    assert all(model.precision[n] == ops.H1 for n in ("local_encoder", "volume_source", "unet3d"))
    src = [c for c in calls if c[0]]
    assert {c[0] for c in src} == set(SOURCE_NETS)
    names = [n for _, n, _, _ in src]
    # the stem: emo_stem_pack, then a 7x1 convolution over its 32 channels, pad (3, 0), with bias and GroupNorm statistics
    assert "emo_conv_direct" not in names and names.count("emo_stem_pack") == 1
    i = names.index("emo_stem_pack")
    assert names[i + 1] == "emo_conv_igemm"
    d = src[i + 1][3][2]
    assert (d.Hin, d.Win, d.Cin, d.kd, d.kh, d.kw, d.ph, d.pw, d.G) == (size, size, 32, 1, 7, 1, 3, 0, 32)
    assert d.bias and d.stats and (d.Hout, d.Wout) == (size, size)
    convs = [c[3] for c in src if c[3] is not None]
    refused = [(k, dry.load().emo_last_error().decode()) for k, (rc, _, _) in enumerate(convs) if rc != 0]
    assert not refused, refused
    assert all(dry.conv_kernel_name(info.kernel).startswith("h1") and info.NP == 1 for _, info, _ in convs)
    assert all(d.operand_fp16 == 1 and not d.a_lo and not d.w_lo for _, _, d in convs)
    assert any(d.kd == 3 for _, _, d in convs) and any(d.Cin == 96 and d.kd == 3 for _, _, d in convs)
    # every one-plane plan written by an apply / post-op in the source networks is one fp16 plane of x16
    applies = [dict(f) for _, n, f, _ in src if n == "emo_apply"]
    assert applies and all(a["plane_fp16"] == 1 and a["plane_scale"] == ops.F16_ACT_SCALE and not a["out_lo"] for a in applies)
    classes = [CP.plan_class(info, d.Din) for _, info, d in convs]
    print(f"\n[fast source pass @{size}^2] {len(convs)} convolutions: "
          + ", ".join(f"{k} x{classes.count(k)}" for k in sorted(set(classes))))
    unswept = sorted(set(classes) - _swept_classes())
    assert not unswept, f"fast-source convolutions in plan classes no GPU case sweeps: {unswept}"


@pytest.mark.parametrize("size", [256, 512])
def test_unswitched_launches_are_unchanged(dry, monkeypatch, size):
    """the identity / expression / head-pose / xy-warp launches of the source pass and every driver-pass launch are the exact
    mode's, descriptor for descriptor (pointers compared by NULL-ness, conv plans by their fields)"""
    _, src_e, drv_e = _record(dry, monkeypatch, size, "exact")
    _, src_f, drv_f = _record(dry, monkeypatch, size, _source_fast())

    def rest(calls):
        return [(n, f, _fields(p[1]) if p else None) for w, n, f, p in calls if not w]

    assert rest(src_f) == rest(src_e)
    assert [(n, f, _fields(p[1]) if p else None) for _, n, f, p in drv_f] == \
        [(n, f, _fields(p[1]) if p else None) for _, n, f, p in drv_e]
    # exact mode: the stem is conv_direct and no source conv is on one plane
    src = [c for c in src_e if c[0]]
    assert [n for _, n, _, _ in src].count("emo_conv_direct") == 1
    assert all(p[1].NP == 2 for _, _, _, p in src if p is not None)


def test_gpu_cases_reach_their_plan_class(dry):
    """the cases of tests/test_fast_source_gpu.py plan as they say at 132 SMs (H100 SXM)"""
    import test_fast_source_gpu as TF
    from emoportraits_b200 import ops

    bad = []
    for want, c in TF.CASES + [TF.DEPTH_CASE]:
        x, w, b, res = TF.make(c, ops, "cpu")
        st = torch.zeros((1, TF.G, 2), dtype=torch.float64) if c.stats else None
        a, pw, kw = TF.conv_args(c, ops, x, w, b, res, st)
        info = ops.conv_plan(a, pw, sm_count=132, **kw)
        if CP.plan_class(info, c.sp[0]) != want or info.NP != 1:
            bad.append((c.id, want, CP.plan_class(info, c.sp[0])))
    assert not bad, bad
    a, pw, kw = TF.conv_args(TF.DEPTH_CASE[1], ops, *TF.make(TF.DEPTH_CASE[1], ops, "cpu"),
                             stats=torch.zeros((1, TF.G, 2), dtype=torch.float64))
    assert ops.conv_plan(a, pw, sm_count=132, **kw).td > 1


# ------------------------------------------------------------------------------------------------------------------
def test_model_accepts_one_plane_source_networks():
    from emoportraits_b200 import ops
    from emoportraits_b200.infer import Model

    assert Model.SOURCE_FAST == dict(local_encoder=ops.H1, volume_source=ops.H1, unet3d=ops.H1)
    pr = Model.resolve_precision(dict(Model.SOURCE_FAST))
    assert pr == dict(Model.PRECISION, **Model.SOURCE_FAST)
    both = Model.resolve_precision(dict(Model.PRESETS["fast"], **Model.SOURCE_FAST))
    assert both == dict(Model.PRECISION, decoder=ops.H1, **Model.SOURCE_FAST)
    for net in ("local_encoder", "volume_source", "unet3d"):
        assert Model.resolve_precision({net: ops.H1})[net] == ops.H1
    assert Model.PRESETS["fast"] == dict(decoder=ops.H1)            # fast mode alone leaves the source pass exact
    for net in ("head_pose", "expression", "idt", "warp"):
        with pytest.raises(ValueError, match="sampler") as e:
            Model.resolve_precision(dict(Model.SOURCE_FAST, **{net: ops.H1}))
        assert net in str(e.value)


def test_inference_wrapper_source_precision_argument():
    from emoportraits_b200.infer import InferenceWrapper

    for bad in ("turbo", "FAST", None, "h1", 1):
        with pytest.raises(ValueError, match="source_precision"):
            InferenceWrapper("x", source_precision=bad)
    with pytest.raises(ValueError, match="precision"):
        InferenceWrapper("x", precision="turbo", source_precision="fast")
    if not torch.cuda.is_available():   # valid settings pass the checks and reach the device requirement
        for pr in ("exact", "fast"):
            with pytest.raises(RuntimeError, match="CUDA"):
                InferenceWrapper("x", precision=pr, source_precision="fast")
