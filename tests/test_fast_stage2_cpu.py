"""CPU tests of stage 2's fast mode (stage2.Stage2Model(precision="fast")):
  * `precision=` of Stage2Model and of the stage-2 InferenceWrapper;
  * in EMO_DRY_RUN mode, at 512^2 batch 1, 1024^2 batch 4 and 1024^2 batch 16 (video.drive_image_with_video's chunk), every
    stage-2 convolution, the stem included, plans on one fp16 plane (NP = 1), none is refused, and each falls in a plan class
    that tests/test_fast_stage2_gpu.py or tests/test_fast_decoder_gpu.py sweeps on the GPU;
  * exact mode issues no one-plane convolution and runs the stem as one emo_conv_direct launch;
  * every case of tests/test_fast_stage2_gpu.py reaches the plan class it names at 132 SMs;
  * the host stem weight is nets.stem_weight's, rearranged; emo_stem_pack refuses every malformed argument."""
import ctypes as C

import pytest
import torch

FAKE = 0x1000   # a 16-byte aligned non-null "device pointer" that is never dereferenced: the calls below are refused first


@pytest.fixture
def dry(monkeypatch):
    from emoportraits_b200 import lib as L

    monkeypatch.setattr(L, "DRY_RUN", True)   # host tensors are accepted as operands; nothing is launched
    return L


def test_stage2_model_precision_argument():
    from emoportraits_b200.stage2 import Stage2Config, Stage2Model

    cfg = Stage2Config(output_size=512)
    for bad in ("turbo", "FAST", None, 2, "h1"):
        with pytest.raises(ValueError, match="precision"):
            Stage2Model(cfg, {}, "cpu", precision=bad)
    with pytest.raises(TypeError):
        Stage2Model(cfg, {}, "cpu", planes=2)      # precision= replaces planes=


def test_stage2_wrapper_precision_argument():
    from emoportraits_b200.stage2 import InferenceWrapper

    for bad in ("turbo", None):
        with pytest.raises(ValueError, match="precision"):
            InferenceWrapper("x", precision=bad)
    if not torch.cuda.is_available():   # a valid setting passes the check and reaches the device requirement
        with pytest.raises(RuntimeError, match="CUDA"):
            InferenceWrapper("x", precision="fast")


def _record_stage2(L, monkeypatch, size, batch, precision):
    """(model, [(C-ABI call name, conv plan or None)]) of one dry-run stage-2 forward; a plan is (return code, ConvPlanInfo,
    emo_conv_desc) at 132 SMs"""
    from emoportraits_b200.stage2 import Stage2Config, Stage2Model, synthetic_state_dict_s2

    lib = L.load()
    calls = []
    launch = L.call

    def call(name, *args):
        plan = None
        if name == "emo_conv_igemm":
            d = args[0]._obj
            info = L.ConvPlanInfo()
            plan = (lib.emo_conv_plan(C.byref(d), 132, C.byref(info)), info, type(d).from_buffer_copy(d))
        calls.append((name, plan))
        return launch(name, *args)

    monkeypatch.setattr(L, "call", call)
    cfg = Stage2Config(output_size=size)
    model = Stage2Model(cfg, synthetic_state_dict_s2(cfg, 0), "cpu", precision=precision)
    model.forward(torch.rand(batch, 3, 512, 512))
    return model, calls


def _swept_classes():
    import test_fast_decoder_gpu as TD
    import test_fast_stage2_gpu as TS

    return {w for w, _ in TD.CASES} | {w for w, _ in TS.CASES}


@pytest.mark.parametrize("size,batch", [(512, 1), (1024, 4), (1024, 16)])
def test_fast_mode_plans_every_stage2_conv_on_one_plane(dry, monkeypatch, size, batch):
    import test_fast_stage2_gpu as TS
    from emoportraits_b200 import ops

    model, calls = _record_stage2(dry, monkeypatch, size, batch, "fast")
    assert model.planes == ops.H1
    names = [n for n, _ in calls]
    assert "emo_conv_direct" not in names and names.count("emo_stem_pack") == 1
    convs = [p for _, p in calls if p is not None]
    refused = [(i, dry.load().emo_last_error().decode()) for i, (rc, _, _) in enumerate(convs) if rc != 0]
    assert not refused, refused
    assert all(info.NP == 1 and info.fp16 == 1 for _, info, _ in convs)
    assert all(d.operand_fp16 == 1 and not d.a_lo and not d.w_lo for _, _, d in convs)
    # the stem: emo_stem_pack, then a 7x1 convolution over its 32 channels, pad (3, 0), with bias, writing fp32 (N,1,S,S,128)
    i = names.index("emo_stem_pack")
    assert names[i + 1] == "emo_conv_igemm"
    d = calls[i + 1][1][2]
    assert (d.N, d.Hin, d.Win, d.Cin, d.Cout, d.kd, d.kh, d.kw, d.ph, d.pw) == (batch, size, size, 32, 128, 1, 7, 1, 3, 0)
    assert d.bias and (d.Hout, d.Wout) == (size, size) and not d.out_nchw
    classes = [TS._plan_class(info) for _, info, _ in convs]
    print(f"\n[fast stage 2 @{size}^2 batch {batch}] {len(convs)} convolutions: "
          + ", ".join(f"{k} x{classes.count(k)}" for k in sorted(set(classes))))
    unswept = sorted(set(classes) - _swept_classes())
    assert not unswept, f"fast-mode stage-2 convolutions in plan classes no GPU case sweeps: {unswept}"


@pytest.mark.parametrize("size,batch", [(512, 1), (1024, 4)])
def test_exact_mode_is_unchanged(dry, monkeypatch, size, batch):
    model, calls = _record_stage2(dry, monkeypatch, size, batch, "exact")
    assert model.planes == 2 and model.stem_h1 is None
    names = [n for n, _ in calls]
    assert names.count("emo_conv_direct") == 1 and "emo_stem_pack" not in names
    convs = [p for _, p in calls if p is not None]
    assert convs and all(rc == 0 and info.NP == 2 and info.fp16 == 0 for rc, info, _ in convs)
    assert all(d.operand_fp16 == 0 and d.a_lo and d.w_lo for _, _, d in convs)


def test_gpu_cases_reach_their_plan_class(dry):
    """the cases of tests/test_fast_stage2_gpu.py plan as they say at 132 SMs (H100 SXM)"""
    import test_fast_stage2_gpu as TS
    from emoportraits_b200 import ops

    bad = []
    for want, c in TS.CASES:
        x, w, b, res, A, B = TS.make(c, ops, "cpu")
        a, pw, kw = TS.conv_args(c, ops, x, w, b, res, A, B)
        info = ops.conv_plan(a, pw, sm_count=132, **kw)
        if TS._plan_class(info) != want:
            bad.append((c.id, want, TS._plan_class(info)))
    assert not bad, bad


def test_stem_weight_is_the_direct_stem_rearranged():
    from emoportraits_b200 import nets, ops
    from emoportraits_b200.stage2 import Stage2Config, synthetic_state_dict_s2

    cfg = Stage2Config(output_size=512)
    wd, _ = nets.stem_weight(synthetic_state_dict_s2(cfg, 0), "local_encoder.from_rgb_512px", "cpu")   # (7, 7, 4, 128)
    pw = ops.pack_stem_weight(wd, device="cpu")
    assert pw.f16 and pw.lo is None and pw.scale == ops.F16_W_SCALE and pw.k == (1, 7, 1)
    assert (pw.cin, pw.cout, pw.cout_pad) == (32, 128, 128) and pw.hi.shape == (7, 128, 32)
    want = torch.zeros(7, 128, 32)
    for ky in range(7):
        for kx in range(7):
            for c in range(4):
                want[ky, :, kx * 4 + c] = wd[ky, kx, c]
    assert torch.equal(pw.hi, (want * ops.F16_W_SCALE).half())
    assert torch.equal(pw.hi[:, :, 28:], torch.zeros(7, 128, 4, dtype=torch.float16))
    assert torch.equal(pw.hi.view(7, 128, 8, 4)[:, :, :7, 3], torch.zeros(7, 128, 7, dtype=torch.float16))   # the padded 4th channel


def test_stem_pack_refuses_bad_arguments():
    from emoportraits_b200 import lib as L

    lib = L.load()
    ok = dict(x=FAKE, N=1, H=8, W=8, C=4, scale=16.0, out=FAKE)
    cases = {
        "null x": dict(x=None), "null out": dict(out=None), "misaligned x": dict(x=FAKE + 4), "misaligned out": dict(out=FAKE + 8),
        "C = 3": dict(C=3), "C = 8": dict(C=8), "N = 0": dict(N=0), "H = 0": dict(H=0), "W < 0": dict(W=-1),
        "scale 0": dict(scale=0.0),
    }
    for name, kw in cases.items():
        a = dict(ok, **kw)
        rc = lib.emo_stem_pack(a["x"], a["N"], a["H"], a["W"], a["C"], a["scale"], a["out"], None)
        assert rc == -1, (name, rc)                                                   # EMO_ERR_INVALID
        assert "emo_stem_pack" in lib.emo_last_error().decode(), name
