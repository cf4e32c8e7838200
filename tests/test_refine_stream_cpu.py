"""CPU tests of refined frames in flight (Stage2Model.refine, Model.make_driver_graph / DriverPipeline with refine=,
InferenceWrapper.forward_refined, emo_s2_prepare / emo_s2_finish):
  * in EMO_DRY_RUN mode, for exact and fast stage 2 at 256^2 -> 512^2 and 512^2 -> 1024^2, a refined frame issues the stage-1
    frame's launches, then emo_s2_prepare, then exactly the eager Stage2Model.forward's launches after its resize (and, fast,
    its stem_pack), descriptor for descriptor, then emo_s2_finish;
  * refine with an encoding frame, a stage-2 model on another device and a u8_out that does not fit are refused before a
    stream is created or anything is queued; so are forward_refined's bad inputs;
  * the two entry points refuse null pointers, bad shapes, a missing or doubled stem operand and a misaligned operand."""
import ctypes as C
from types import SimpleNamespace

import pytest
import torch

from test_embedding_drive_cpu import _bare_pipeline, _identity
from test_embedding_drive_cpu import _wrapper as _host_wrapper
from test_identity_switch_cpu import _model, _recorder

FAKE = 0x1000   # a 16-byte aligned non-null "device pointer" that is never dereferenced: the calls below are refused first


@pytest.fixture
def dry(monkeypatch):
    from emoportraits_b200 import lib as L

    monkeypatch.setattr(L, "DRY_RUN", True)   # host tensors are accepted as operands; nothing is launched
    return L


def _stage2(size, precision):
    from emoportraits_b200.stage2 import Stage2Config, Stage2Model, synthetic_state_dict_s2

    cfg = Stage2Config(output_size=size)
    return Stage2Model(cfg, synthetic_state_dict_s2(cfg, 0), "cpu", precision=precision)


def _launches(calls, fn):
    calls.clear()
    fn()
    return list(calls)


@pytest.mark.parametrize("precision", ["exact", "fast"])
@pytest.mark.parametrize("size,s2_size", [(256, 512), (512, 1024)])
def test_refined_frame_launch_sequence(dry, monkeypatch, size, s2_size, precision):
    _, model = _model(size)
    s2 = _stage2(s2_size, precision)
    torch.manual_seed(0)
    x = torch.rand(1, 3, size, size)
    st = model.source_pass(x)
    calls, _ = _recorder(dry, monkeypatch)
    frame = _launches(calls, lambda: model.driver_pass(st, x, mix=True))
    img = torch.rand(1, 3, size, size)
    eager = _launches(calls, lambda: s2.forward(img))
    refined = _launches(calls, lambda: s2.refine(model.driver_pass(st, x, mix=True)[0]))
    # the eager stage 2 starts with the resize (and, fast, the stem's plane): the prepare pass replaces them
    skip = ["emo_resize_bilinear"] + (["emo_stem_pack"] if precision == "fast" else [])
    assert [c[0] for c in eager[:len(skip)]] == skip
    body = eager[len(skip):]
    assert refined[:len(frame)] == frame
    prep, fin = refined[len(frame)], refined[-1]
    assert refined[len(frame) + 1:-1] == body
    fast = precision == "fast"
    assert prep == ("emo_s2_prepare", ("ptr", 1, size, size, s2_size, "ptr", None if fast else "ptr", "ptr" if fast else None,
                                       16.0 if fast else 0.0, 0)), prep
    assert fin == ("emo_s2_finish", ("ptr", "ptr", 1, s2_size, s2_size, "ptr", "ptr", 0)), fin
    assert not {"emo_image_to_u8", "emo_resize_bilinear", "emo_stem_pack"} & {c[0] for c in refined[len(frame):]}


def test_refine_outputs_in_place(dry):
    s2 = _stage2(512, "exact")
    out, u8 = torch.empty(2, 3, 512, 512), torch.empty(2, 512, 512, 3, dtype=torch.uint8)
    resized, ffhq, got = s2.refine(torch.rand(2, 3, 256, 256), out=out, u8=u8)
    assert ffhq is out and got is u8 and resized.shape == (2, 3, 512, 512)
    with pytest.raises(AssertionError):
        s2.refine(torch.rand(1, 3, 256, 256), u8=torch.empty(1, 512, 512, 4, dtype=torch.uint8))


# ---- what a refining pipeline refuses ---------------------------------------------------------------------------------------
def _checker(device="cpu"):
    """a stand-in for Model with its two input checks (DriverPipeline calls them before it creates a stream)"""
    from emoportraits_b200.infer import Model

    m = SimpleNamespace(device=torch.device(device), check_inputs=Model.check_inputs)
    m.check_refine = lambda refine, encode: Model.check_refine(m, refine, encode)
    return m


def test_refine_is_refused_with_encode_and_across_devices():
    from emoportraits_b200.infer import DriverPipeline

    m = _checker()
    here, there = SimpleNamespace(device=torch.device("cpu")), SimpleNamespace(device=torch.device("cuda", 1))
    m.check_refine(None, True)
    m.check_refine(here, False)
    with pytest.raises(ValueError, match="encod"):
        m.check_refine(here, True)
    with pytest.raises(ValueError, match="device"):
        m.check_refine(there, False)
    for kw in (dict(encode=True, refine=here), dict(refine=there)):
        with pytest.raises(ValueError):
            DriverPipeline(m, None, depth=4, **kw)


def test_submit_refuses_bad_u8_out():
    from emoportraits_b200.config import shipped_config
    from emoportraits_b200.stage2 import Stage2Config

    cfg = shipped_config(256)
    img = torch.zeros(1, 3, 256, 256)
    refine = SimpleNamespace(cfg=Stage2Config(output_size=512))
    u8 = lambda *shape: torch.zeros(*shape, dtype=torch.uint8)   # noqa: E731
    cases = [(None, u8(1, 512, 512, 3)),                                       # not a refining pipeline
             (refine, u8(1, 256, 256, 3)), (refine, u8(512, 512, 3)), (refine, u8(2, 512, 512, 3)),
             (refine, torch.zeros(1, 512, 512, 3)), (refine, u8(1, 3, 512, 512)),
             (refine, u8(1, 512, 3, 512).transpose(2, 3)), (refine, [0] * 3)]
    for r, bad in cases:
        pipe = _bare_pipeline(cfg, refine=r)
        st0 = pipe.st
        with pytest.raises(ValueError, match="u8_out"):
            pipe.submit(img, u8_out=bad, st=SimpleNamespace(**vars(_identity(cfg))))
        assert pipe.n == 0 and pipe.st is st0


# ---- forward_refined ----------------------------------------------------------------------------------------------------
def _s2_wrapper(device="cpu", size=512, precision="exact"):
    from emoportraits_b200.stage2 import Stage2Config

    return SimpleNamespace(model_two=SimpleNamespace(device=torch.device(device), cfg=Stage2Config(output_size=size),
                                                     precision=precision))


def _refining_wrapper(monkeypatch, state=True):
    w = _host_wrapper(state=state)
    w.model = _checker()
    seen = []

    def pipeline(mix, target_theta, mix_old, refine=None, **inputs):
        seen.append(dict(mix=mix, target_theta=target_theta, mix_old=mix_old, refine=refine, **inputs))
        return SimpleNamespace(refine=refine, depth=4)

    monkeypatch.setattr(w, "_driver_pipeline", pipeline)
    monkeypatch.setattr(w, "_render", lambda pipe, n, inputs: seen.append((pipe, [inputs(i) for i in range(n)])))
    return w, seen


def test_forward_refined_refuses_before_queueing(monkeypatch):
    w, seen = _refining_wrapper(monkeypatch)
    E = w.cfg.expr_channels
    s2 = _s2_wrapper()
    frames = torch.rand(2, 3, 256, 256)
    three = lambda n: (torch.ones(n, 3), torch.zeros(n, 3), torch.zeros(n, 3))   # noqa: E731
    bad = [
        dict(driver_images=frames, inferer_s2=object()),                                       # not a stage-2 wrapper
        dict(driver_images=frames, inferer_s2=_s2_wrapper(torch.device("cuda", 1))),           # another device
        dict(driver_images=None, inferer_s2=s2),                                              # neither images nor embeddings
        dict(driver_images=None, inferer_s2=s2, custome_target_theta_embed=three(2)),
        dict(driver_images=None, inferer_s2=s2, custome_target_pose_embed=torch.zeros(2, E)),
        dict(driver_images=None, inferer_s2=s2, custome_target_theta_embed=three(2), custome_target_pose_embed=torch.zeros(3, E)),
        dict(driver_images=None, inferer_s2=s2, custome_target_theta_embed=three(2), custome_target_pose_embed=torch.zeros(2, E + 1)),
        dict(driver_images=None, inferer_s2=s2, custome_target_theta_embed=(torch.ones(2, 9),), custome_target_pose_embed=torch.zeros(2, E)),
        dict(driver_images=frames, inferer_s2=s2, custome_target_theta_embed=three(2)),    # one pose for every frame
        dict(driver_images=frames, inferer_s2=s2, custome_target_pose_embed=torch.zeros(E + 1)),
        dict(driver_images=[], inferer_s2=s2),
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            w.forward_refined(**kw)
    with pytest.raises(TypeError):
        w.forward_refined(frames, s2, smooth_pose=True)                                    # a recurrence: no such form
    none, seen_none = _refining_wrapper(monkeypatch, state=False)
    with pytest.raises(RuntimeError, match="source"):
        none.forward_refined(frames, s2)
    assert not seen and not seen_none


def test_forward_refined_queues_frames_on_a_refining_pipeline(monkeypatch):
    w, seen = _refining_wrapper(monkeypatch)
    E = w.cfg.expr_channels
    s2 = _s2_wrapper()
    frames = torch.rand(3, 3, 256, 256)
    w.forward_refined(frames, s2, mix=True, mix_old=False)
    flags, (pipe, subs) = seen[0], seen[1]
    assert flags == dict(mix=True, target_theta=True, mix_old=False, refine=s2.model_two, theta_embed=False, pose_embed=False)
    assert pipe.refine is s2.model_two and len(subs) == 3
    assert all(torch.equal(s["drv"], frames[i:i + 1]) and s["theta_embed"] is None and s["pose_embed"] is None
               for i, s in enumerate(subs))
    seen.clear()
    theta = (torch.ones(4, 3), torch.full((4, 3), 0.1), torch.full((4, 3), 0.2))
    pe = torch.rand(4, E)
    w.forward_refined(None, s2, custome_target_theta_embed=theta, custome_target_pose_embed=pe)
    flags, (_, subs) = seen[0], seen[1]
    assert flags["refine"] is s2.model_two and flags["image"] is False and flags["theta_embed"] and flags["pose_embed"]
    assert len(subs) == 4 and all(s["drv"] is None for s in subs)
    assert torch.equal(torch.cat([s["theta_embed"] for s in subs]), torch.cat(theta, 1))
    assert torch.equal(torch.cat([s["pose_embed"] for s in subs]), pe)


# ---- the entry points' argument checks ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    from emoportraits_b200 import lib as L

    if L.DRY_RUN:
        pytest.skip("EMO_DRY_RUN skips the calls")
    L.load()
    return L


def _refused(lib, rc, match):
    assert rc == -1, rc                                  # EMO_ERR_INVALID
    msg = lib.emo_last_error().decode()
    assert match in msg, msg


def test_s2_prepare_guards(L):
    lib = L.load()
    f = lambda *a: lib.emo_s2_prepare(*a, None)   # noqa: E731
    _refused(lib, f(None, 1, 256, 256, 512, FAKE, FAKE, None, 0.0), "null pointer")
    _refused(lib, f(FAKE, 1, 256, 256, 512, None, FAKE, None, 0.0), "null pointer")
    _refused(lib, f(FAKE, 1, 256, 256, 512, FAKE, None, None, 0.0), "exactly one stem operand")
    _refused(lib, f(FAKE, 1, 256, 256, 512, FAKE, FAKE, FAKE, 16.0), "exactly one stem operand")
    for shape in ((0, 256, 256, 512), (1, 0, 256, 512), (1, 256, 0, 512), (1, 256, 256, 0)):
        _refused(lib, f(FAKE, *shape, FAKE, FAKE, None, 0.0), "bad shape")
    _refused(lib, f(FAKE, 1, 256, 256, 512, FAKE, None, FAKE + 8, 16.0), "16-byte aligned")
    _refused(lib, f(FAKE, 1, 256, 256, 512, FAKE, FAKE + 4, None, 0.0), "16-byte aligned")
    _refused(lib, f(FAKE, 1, 256, 256, 512, FAKE, None, FAKE, 0.0), "plane_scale")
    _refused(lib, f(FAKE, 1 << 20, 256, 256, 1 << 12, FAKE, FAKE, None, 0.0), "grid too large")


def test_s2_finish_guards(L):
    lib = L.load()
    f = lambda *a: lib.emo_s2_finish(*a, None)    # noqa: E731
    for k in range(4):
        ptrs = [FAKE] * 4
        ptrs[k] = None
        _refused(lib, f(ptrs[0], ptrs[1], 1, 512, 512, ptrs[2], ptrs[3]), "null pointer")
    for shape in ((0, 512, 512), (1, 0, 512), (1, 512, 0)):
        _refused(lib, f(FAKE, FAKE, *shape, FAKE, FAKE), "bad shape")
